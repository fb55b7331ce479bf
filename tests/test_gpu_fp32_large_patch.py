"""The fp32 CUDA-core engine (UDH_NUMERIC_FP32) across its whole patch range, up to P = 1408.

Above P = 128 this engine is the only mode, and check_cnn_args accepts any multiple of 128 up to 1408.  From P = 1152 on, fc1's
weights, weight gradient and Adam moments, F x 1024 with F = (P/8)^2 128, have elements past index 2^31, where an `int` offset
would wrap; the convolutions run at spatial sizes up to 1408.  test_gpu_fp32_certify.py certifies P = 128 and 256; this file
holds the rest of the range to the same standard:
  1. every conv / dgrad / weight-gradient / pool instance of the step at its size for P = 384 and 640 (odd multiples of 128:
     conv4 at 48 and 80 pixels, an odd count of 16-wide tiles) and P = 1408, B = 1 and 2 (B = 1 at 640): exact integer
     operands equal float64, forward and dgrad equal their restated fmaf chain on sampled tiles (the last tile of the last image
     included), every element within its gamma bound of a float64 reference computed in row bands on the device;
  2. fc1's three GEMMs through udh_debug_fc1_ex at P = 1024, 1152 and 1408 (F x 1024 = 2^31, 2.7e9 and 4.1e9 weights), B = 1, 2
     and 3: exact operands, y and dx within the gamma bound of their chains, dW at B = 1 bit-identical to fl(x dy) on every
     element, and the worst element reported separately past flat index 2^31 and in the last 64-row CTA row of dW;
  3. udh_adam_step over the whole 4.06e9-float flat buffer of P = 1408: per-element bound on stripes across 2^31 bytes, 2^32
     bytes and 2^31 floats, on the tail and on a random sample; the guard bands untouched; grid caps 1 and the default
     bit-identical;
  4. the engine at P = 384 (B = 1, 2) and 1408 (B = 1): forward layer by layer against float64 on its own inputs with pools
     exact, udh_cnn_bwd against a float64 backward on its own gates, and one h_loss step: pred_h4p against a float64 forward
     and Adam's update of sampled fc1 weights past 2^31;
  5. the TF checkpoint and the .pt state_dict of a P = 1152 engine (a 10.9 GB fc1 tensor) round-trip bit for bit.
Every case computes the device (and host) memory it needs, its own buffers included, and skips, printing need and free, when
the card cannot hold it; the large cases release their buffers on failure, so one failure does not make the next ones skip."""
import os
import shutil
import tempfile
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import optim as OPT                                              # noqa: E402
from oracle import simt_fp32 as S                                            # noqa: E402
from _pool_ties import tie_windows                                           # noqa: E402
from _fp32_simt import (CONVS, DGRADS, POOLS, P_, acts, band_rows, check_bound, check_chain, check_conv_banded,  # noqa: E402
                        check_exact, check_pool, cnn_fwd, conv_params, flat_batch, image_size, int_tensor, layer_input,
                        ref_conv_rows, ref_wgrad_banded, simt_conv, simt_wgrad)

GiB = float(1 << 30)
LAYER_BATCHES = [(1, 384), (2, 384), (1, 640), (1, 1408), (2, 1408)]
FC1_PATCHES = [1024, 1152, 1408]
ROWS = 1 << 16                    # fc1 weight rows per chunk of the float64 checks (64 M elements)
TWO31 = 1 << 31


@pytest.fixture(scope="module")
def udh():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from unsuperviseddeephomographyral2018_b200 import _lib, engine, ops, params
    _lib.require_device()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False

    class NS:
        pass
    ns = NS()
    ns.lib, ns.ops, ns.engine, ns.params, ns.L = _lib, ops, engine, params, _lib.lib
    yield ns
    torch.cuda.empty_cache()


def _ids(v):
    return "B%d-P%d" % v


def need_device(nbytes, what):
    """Skip unless the device has nbytes free (plus 1 GiB of slack for the library's scratch and the allocator)."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    if free < nbytes + GiB:
        pytest.skip("%s needs %.1f GiB of device memory (+1 GiB slack), %.1f of %.1f GiB free" % (what, nbytes / GiB, free / GiB, total / GiB))
    print("%s: needs %.1f GiB of device memory, %.1f of %.1f GiB free" % (what, nbytes / GiB, free / GiB, total / GiB))


def host_available():
    with open("/proc/meminfo") as f:
        for ln in f:
            if ln.startswith("MemAvailable:"):
                return int(ln.split()[1]) * 1024
    return 0


def need_host(nbytes, what):
    avail = host_available()
    if avail < nbytes:
        pytest.skip("%s needs %.1f GiB of host memory, %.1f GiB available" % (what, nbytes / GiB, avail / GiB))
    print("%s: needs %.1f GiB of host memory, %.1f GiB available" % (what, nbytes / GiB, avail / GiB))


def release(*tensors):
    """Free the device memory of tensors now, views included: a failed assertion's traceback keeps the test's frames (and so
    its buffers) alive, and the next large case would otherwise skip for memory instead of running."""
    for t in tensors:
        t.untyped_storage().resize_(0)


def release_engine(eng):
    release(eng.params, eng.grads, eng.adam_m, eng.adam_v, eng.ws)


def feat(Pz):
    return (Pz // 8) ** 2 * 128


# ------------------------------------------------------------------------------------------------ 1. layer kernels
def _layer_need(B, H, cin, cout):
    """Device bytes of one layer case: inputs and outputs in fp32 (x, out, a mask / gradient of the same size, the restated
    gathers), plus float64 row bands of the reference and its bound."""
    return 4 * B * H * H * (2 * cin + 3 * cout) + 12 * 8 * (1 << 25)


@pytest.mark.parametrize("name,div,cin,cout", CONVS)
@pytest.mark.parametrize("BP", LAYER_BATCHES, ids=_ids)
def test_conv_forward_large(udh, BP, name, div, cin, cout):
    B, Pz = BP
    H = Pz // div
    need_device(_layer_need(B, H, cin, cout), "%s forward B=%d P=%d" % (name, B, Pz))
    t0 = time.time()
    seed = B * 1000 + Pz + H + cin
    two = cin == 2
    g = torch.Generator(device="cuda").manual_seed(seed)
    what = "fp32 %s forward B=%d P=%d" % (name, B, Pz)
    split = lambda x: (x[..., :1].contiguous(), x[..., 1:].contiguous()) if two else (x, None)
    x = int_tensor(g, (B, H, H, cin)); w = int_tensor(g, (3, 3, cin, cout)); b = int_tensor(g, (cout,), -3, 3)
    x1, x2 = split(x)
    check_conv_banded(simt_conv(udh, x1, w, b, relu=1, x2=x2), x, w, b, False, what + " (exact operands)", relu=True, exact=True)
    x = torch.randn(B, H, H, cin, device="cuda", generator=g)
    w = (torch.randn(3, 3, cin, cout, device="cuda", generator=g) / (3 * cin ** 0.5)).contiguous()
    b = (torch.randn(cout, device="cuda", generator=g) * 0.1).contiguous()
    x1, x2 = split(x)
    for relu in (1, 0):
        out = simt_conv(udh, x1, w, b, relu=relu, x2=x2)
        n = check_chain(out, x1, w, b, None, relu, False, seed + relu, what + (" relu" if relu else " linear"), x2=x2)
        frac = check_conv_banded(out, x, w, b, False, what, relu=bool(relu))
        del out
        print("%s relu=%d: exact operands equal, %d restated chains equal, max err %.3f of gamma_{K+1} bound (%.1f s)"
              % (what, relu, n, frac, time.time() - t0))


@pytest.mark.parametrize("name,div,cin,cout,masked", DGRADS)
@pytest.mark.parametrize("BP", LAYER_BATCHES, ids=_ids)
def test_dgrad_large(udh, BP, name, div, cin, cout, masked):
    B, Pz = BP
    H = Pz // div
    need_device(_layer_need(B, H, cin, cout), "%s dgrad B=%d P=%d" % (name, B, Pz))
    t0 = time.time()
    seed = B * 1000 + Pz + H + cin + 7 * masked
    gen = torch.Generator(device="cuda").manual_seed(seed)
    what = "fp32 %s dgrad%s B=%d P=%d" % (name, " + mask" if masked else "", B, Pz)
    gi = int_tensor(gen, (B, H, H, cout)); w = int_tensor(gen, (3, 3, cin, cout))
    mask = int_tensor(gen, (B, H, H, cin), -1, 2) if masked else None
    check_conv_banded(simt_conv(udh, gi, w, mask=mask, dgrad=1), gi, w, None, True, what + " (exact operands)", mask=mask, exact=True)
    gi = (torch.randn(B, H, H, cout, device="cuda", generator=gen) * 0.1).contiguous()
    w = (torch.randn(3, 3, cin, cout, device="cuda", generator=gen) / (3 * cin ** 0.5)).contiguous()
    mask = F.relu(torch.randn(B, H, H, cin, device="cuda", generator=gen)).contiguous() if masked else None
    out = simt_conv(udh, gi, w, mask=mask, dgrad=1)
    n = check_chain(out, gi, w, None, mask, False, True, seed, what)
    if masked:
        assert (out[mask <= 0] == 0).all(), what
    frac = check_conv_banded(out, gi, w, None, True, what, mask=mask)
    print("%s: exact operands equal, %d restated chains equal, max err %.3f of gamma_{K+1} bound (%.1f s)" % (what, n, frac, time.time() - t0))


@pytest.mark.parametrize("name,div,cin,cout", CONVS)
@pytest.mark.parametrize("BP", LAYER_BATCHES, ids=_ids)
def test_wgrad_large(udh, BP, name, div, cin, cout):
    B, Pz = BP
    H = Pz // div
    need_device(_layer_need(B, H, cin, cout), "%s wgrad B=%d P=%d" % (name, B, Pz))
    t0 = time.time()
    seed = B * 77 + Pz + H + cin
    gen = torch.Generator(device="cuda").manual_seed(seed)
    two = cin == 2
    what = "fp32 %s wgrad B=%d P=%d" % (name, B, Pz)
    split = lambda x: (x[..., :1].contiguous(), x[..., 1:].contiguous()) if two else (x, None)
    x = int_tensor(gen, (B, H, H, cin)); go = int_tensor(gen, (B, H, H, cout))
    x1, x2 = split(x)
    dW, db, part = simt_wgrad(udh, x1, go, cin, x2=x2)
    rW, rb = ref_wgrad_banded(x, go)
    aW, ab = ref_wgrad_banded(x, go, absolute=True)
    assert aW.max() < 2 ** 24 and ab.max() < 2 ** 24, (aW.max().item(), ab.max().item())     # every partial sum stays exact
    check_exact(dW, rW, what + " dW (exact operands)", "ky,kx,ci,co")
    check_exact(db, rb, what + " db (exact operands)", "co")
    ctas, per, rs = part
    tiles = B * (H // 8) * (H // 16)
    assert ctas * per >= tiles > (ctas - 1) * per, part                # the partition covers every tile once
    x = torch.randn(B, H, H, cin, device="cuda", generator=gen)
    go = (torch.randn(B, H, H, cout, device="cuda", generator=gen) * 0.1).contiguous()
    x1, x2 = split(x)
    dW, db, part = simt_wgrad(udh, x1, go, cin, x2=x2)
    rW, rb = ref_wgrad_banded(x, go)
    aW, ab = ref_wgrad_banded(x, go, absolute=True)
    L, m = per * (8 // rs) * 16, ctas * rs
    g_ = float(S.gamma(L + m - 1))
    fW = check_bound(dW, rW, g_ * aW, what + " dW", "ky,kx,ci,co")
    fb = check_bound(db, rb, g_ * ab, what + " db", "co")
    print("%s: partition %d CTAs x %d tiles x %d row phases; exact operands equal; dW %.2e, db %.2e of gamma_{L+m-1} bound (%.1f s)"
          % (what, ctas, per, rs, fW, fb, time.time() - t0))


@pytest.mark.parametrize("name,div,C", POOLS)
@pytest.mark.parametrize("BP", LAYER_BATCHES, ids=_ids)
def test_pool_large(udh, BP, name, div, C):
    B, Pz = BP
    H = Pz // div
    need_device(4 * B * H * H * C * 12, "%s B=%d P=%d" % (name, B, Pz))
    gen = torch.Generator(device="cuda").manual_seed(B * 31 + H + C)
    x = tie_windows(gen, B, H, H, C)
    dout = torch.randn(B, H // 2, H // 2, C, device="cuda", generator=gen)
    dout[..., 0] = -0.0
    ties, zeros = check_pool(udh, x, dout, "fp32 %s B=%d P=%d" % (name, B, Pz))
    windows = B * (H // 2) ** 2 * C
    assert ties > windows // 3 and zeros > windows // 10, (ties, zeros, windows)
    print("fp32 %s B=%d P=%d: forward and routing bit-identical to the rule on %d windows (%d tied positive maxima, %d zero)"
          % (name, B, Pz, windows, ties, zeros))


# ------------------------------------------------------------------------------------------------ 2. fc1 at large F
def fc1_ex(udh, x, w, dy, dW, Pz):
    """udh_debug_fc1_ex -> y, dx (dW accumulated into the caller's zeroed buffer).  y and dx start as NaN."""
    B = x.shape[0]
    y = torch.full((B, 1024), float("nan"), device="cuda")
    dx = torch.full((B, feat(Pz)), float("nan"), device="cuda")
    rc = udh.L.udh_debug_fc1_ex(P_(x), P_(w), P_(dy), P_(y), P_(dW), P_(dx), B, Pz, None)
    assert rc == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    return y, dx


def fwd_split(Fn, B):
    """(k_chunk, splits) of fc1_fwd_simt's split-K SGEMM: K = F cut into 16 chunks (4 above B = 256) of a multiple of 16."""
    s = 16 if B <= 256 else 4
    k_chunk = ((Fn + s - 1) // s + 15) // 16 * 16
    return k_chunk, (Fn + k_chunk - 1) // k_chunk


CHUNK = 1 << 28          # floats per chunk of the whole-buffer fills and comparisons (1 GiB)


def _fill_chunks(t, fn):
    flat = t.view(-1)
    for a in range(0, flat.numel(), CHUNK):
        fn(flat[a:a + CHUNK])


def assert_same_bits(got, want, what):
    """got (a flat buffer) equals want(a, b) on [a, b) bit for bit, one CHUNK at a time (bounded temporaries); want is called
    on consecutive chunks in order, so it may regenerate a seeded stream."""
    flat = got.view(-1)
    for a in range(0, flat.numel(), CHUNK):
        b = min(flat.numel(), a + CHUNK)
        w = want(a, b)
        bad = flat[a:b].view(torch.int32) != w.view(torch.int32)
        if bad.any():
            i = a + bad.nonzero()[0].item()
            pytest.fail("%s: %d elements of [%d, %d) differ, first at %d" % (what, int(bad.sum()), a, b, i))
        del w, bad


class Worst:
    """Largest fraction of the bound over all elements, over rows past flat index 2^31 and over the last 64-row CTA row."""
    def __init__(self):
        self.all = self.hi = self.last = 0.0

    def add(self, frac_rows, r0, Fn, row_elems=1024):
        """frac_rows: per-row worst fraction of a chunk starting at row r0."""
        r = torch.arange(r0, r0 + frac_rows.numel(), device=frac_rows.device)
        self.all = max(self.all, frac_rows.max().item())
        hi = frac_rows[r * row_elems >= TWO31]
        if hi.numel():
            self.hi = max(self.hi, hi.max().item())
        last = frac_rows[r >= Fn - 64]
        if last.numel():
            self.last = max(self.last, last.max().item())

    def __str__(self):
        return "%.2e (past 2^31: %.2e, last CTA row: %.2e)" % (self.all, self.hi, self.last)


def _frac(d, bound, what, r0, names):
    bad = d > bound
    if bad.any():
        i = bad.flatten().nonzero()[0].item()
        r, c = divmod(i, d.shape[1])
        pytest.fail("%s: %d elements over the bound, first at (%s) = (%d, %d): err %.3e > %.3e"
                    % (what, int(bad.sum()), names, r0 + r, c, d.flatten()[i].item(), bound.flatten()[i].item()))
    return torch.where(bound > 0, d / bound.clamp_min(1e-300), (d > 0).double()).amax(dim=1)


@pytest.mark.parametrize("B", [1, 2, 3])
@pytest.mark.parametrize("Pz", FC1_PATCHES)
def test_fc1_large_feature_count(udh, Pz, B):
    """y = x.W, dx = dy.W^T and dW += x^T.dy at F = (P/8)^2 128 through the step's own SIMT calls.  Exact operands first (all
    three outputs equal float64), then real values: y within gamma_{k_chunk + splits} |x| |W| per output (each split an fmaf
    chain of k_chunk terms, the partials added in order), dx within gamma_1024 |dy| |W|^T, dW at B = 1 bit-identical to
    fl(x dy) on all F x 1024 elements and at B = 2, 3 within gamma_B |x|^T |dy|.  Checked in 64 K-row chunks of W on the device.
    W and dW sit in one allocation behind a 2^31-float NaN pad: an element offset that wrapped through a 32-bit int would land
    at most 2^31 floats below its buffer, so it reads the NaN pad (or writes into W) and fails a check, instead of touching
    memory outside the test's allocation."""
    Fn = feat(Pz)
    nW = Fn * 1024
    pad = TWO31
    need_device(4 * (pad + 2 * nW) + 8 * 8 * ROWS * 1024 + 3 * 4 * B * Fn, "fc1 F=%d B=%d" % (Fn, B))
    t0 = time.time()
    g = torch.Generator(device="cuda").manual_seed(Pz * 10 + B)
    arena = torch.empty(pad + 2 * nW, device="cuda")
    try:
        arena[:pad].fill_(float("nan"))
        _fc1_case(udh, Pz, B, arena[pad:pad + nW].view(Fn, 1024), arena[pad + nW:].view(Fn, 1024).zero_(), g, t0)
    finally:
        release(arena)


def _fc1_case(udh, Pz, B, W, dW, g, t0):
    Fn = W.shape[0]
    nW = Fn * 1024
    k_chunk, splits = fwd_split(Fn, B)
    gy, gx, gw = float(S.gamma(k_chunk + splits)), float(S.gamma(1024)), float(S.gamma(B))
    report = {}
    for exact in (True, False):
        if exact:
            _fill_chunks(W, lambda t: t.random_(0, 5, generator=g).sub_(2))
            x, dy = int_tensor(g, (B, Fn)), int_tensor(g, (B, 1024))
        else:
            _fill_chunks(W, lambda t: t.normal_(0.0, 0.01, generator=g))
            x = torch.randn(B, Fn, device="cuda", generator=g).clamp_min(0).contiguous()
            dy = (torch.randn(B, 1024, device="cuda", generator=g) * torch.logspace(-4, -1, B, device="cuda")[:, None]).contiguous()
            dW.zero_()
        y, dx = fc1_ex(udh, x, W, dy, dW, Pz)
        what = "fc1 P=%d F=%d B=%d%s" % (Pz, Fn, B, " (exact operands)" if exact else "")
        assert torch.isfinite(y).all(), what + ": non-finite y"
        assert torch.isfinite(dx).all(), what + ": non-finite dx"
        x64, dy64 = x.double(), dy.double()
        y64 = torch.zeros(B, 1024, dtype=torch.float64, device="cuda")
        ya = torch.zeros_like(y64)
        wx, wW = Worst(), Worst()
        for r0 in range(0, Fn, ROWS):
            r1 = min(Fn, r0 + ROWS)
            Wc = W[r0:r1].double()
            y64 += x64[:, r0:r1] @ Wc
            # dx columns r0..r1 read W rows r0..r1 (flat offset r 1024)
            ref = dy64 @ Wc.T
            if exact:
                check_exact(dx[:, r0:r1], ref, what + " dx", "b,f", off=(0, r0))
            else:
                ya += x64[:, r0:r1].abs() @ Wc.abs()
                dd, bd = (dx[:, r0:r1].double() - ref).abs(), gx * (dy64.abs() @ Wc.abs().T)
                if (dd > bd).any():
                    b_, f_ = divmod((dd > bd).flatten().nonzero()[0].item(), r1 - r0)
                    pytest.fail("%s dx: %d elements over the bound, first at (b,f) = (%d, %d): err %.3e > %.3e"
                                % (what, int((dd > bd).sum()), b_, r0 + f_, dd[b_, f_].item(), bd[b_, f_].item()))
                wx.add((dd / bd.clamp_min(1e-300)).amax(dim=0), r0, Fn)         # dx column f reads W row f
                del dd, bd
            del Wc, ref
            # dW rows r0..r1
            got = dW[r0:r1]
            if exact:
                check_exact(got, x64[:, r0:r1].T @ dy64, what + " dW", "f,o", off=(r0, 0))
            elif B == 1:
                want = x[0, r0:r1, None] * dy[0, None, :]                    # fl(x dy): one product per element,
                want = torch.where(want == 0, torch.zeros_like(want), want)   # fmaf(x, dy, +0) and +0 + that: a zero is +0
                bad = got.view(torch.int32) != want.view(torch.int32)
                if bad.any():
                    i = bad.flatten().nonzero()[0].item()
                    pytest.fail("%s dW: %d elements differ from fl(x dy), first at (f,o) = (%d, %d): %r vs %r"
                                % (what, int(bad.sum()), r0 + i // 1024, i % 1024, got.flatten()[i].item(), want.flatten()[i].item()))
                wW.add(torch.zeros(r1 - r0, device="cuda", dtype=torch.float64), r0, Fn)
            else:
                ref = x64[:, r0:r1].T @ dy64
                wW.add(_frac((got.double() - ref).abs(), gw * (x64[:, r0:r1].abs().T @ dy64.abs()), what + " dW", r0, "f,o"), r0, Fn)
        if exact:
            check_exact(y, y64, what + " y", "b,o")
        else:
            fy = _frac((y.double() - y64).abs(), gy * ya, what + " y", 0, "b,o").max().item()
            report = dict(y=fy, dx=str(wx), dW=("bit-identical to fl(x dy)" if B == 1 else str(wW)))
        del y, dx
    print("fc1 P=%d F=%d (%d weights, %s 2^31) B=%d, splits %d x %d: exact operands equal; y %.2e of gamma_{%d}, dx %s of "
          "gamma_1024, dW %s%s (%.1f s)" % (Pz, Fn, nW, ">" if nW > TWO31 else "=" if nW == TWO31 else "<", B, splits, k_chunk,
                                             report["y"], k_chunk + splits, report["dx"], report["dW"],
                                             "" if B == 1 else " of gamma_%d" % B, time.time() - t0))


# ------------------------------------------------------------------------------------------------ 3. Adam past 2^31 floats
GUARD = 1024          # floats of each guard band (16-byte aligned on both sides)
SENTINEL = 12345.0


def _adam_fill(bufs, n, seed):
    """Seeded p, g, m, v over [GUARD, GUARD + n) in chunks (so the fill can be repeated), guard bands at SENTINEL.  The
    moments are a mid-training state: |g| over nine decades, m of either sign, v >= 0 around g^2 and around eps^2."""
    p, g, m, v = bufs
    for t in bufs:
        t[:GUARD].fill_(SENTINEL); t[GUARD + n:].fill_(SENTINEL)
    C = 1 << 27
    for k, a in enumerate(range(0, n, C)):
        b = min(n, a + C)
        gen = torch.Generator(device="cuda").manual_seed(seed * 100003 + k)
        sl = slice(GUARD + a, GUARD + b)
        p[sl].normal_(0.0, 0.05, generator=gen)
        gg = g[sl]
        gg.normal_(generator=gen)
        gg.mul_(torch.pow(10.0, torch.empty(b - a, device="cuda").uniform_(-9.0, 0.0, generator=gen)))
        m[sl].uniform_(-1.0, 1.0, generator=gen).mul_(gg)
        v[sl].uniform_(0.5, 2.0, generator=gen).mul_(gg).mul_(gg).add_(1e-16)


def _digest(t, n, weights):
    """Position-weighted int64 sum of the bit patterns of t[GUARD : GUARD + n] per chunk: any single-element difference
    changes it (odd weights)."""
    out, C = [], weights.numel()
    for a in range(0, n, C):
        b = min(n, a + C)
        out.append((t[GUARD + a:GUARD + b].view(torch.int32).long() * weights[:b - a]).sum().item())
    return out


def test_adam_whole_buffer_past_2_31(udh):
    """udh_adam_step over the P = 1408 flat buffer (about 4.06e9 floats, 1.0e9 float4s): every checked element within
    oracle.optim.adam_bound of the float64 update, the guard bands untouched, grid caps 1 and 0 (the default) bit-identical."""
    n = udh.L.udh_param_total_floats(1408)
    assert n > TWO31 and n % 4 == 0
    C = 1 << 26
    need_device(4 * 4 * (n + 2 * GUARD) + 8 * C * 3 + 4 * (1 << 27) * 2, "Adam over %d floats" % n)
    t0 = time.time()
    bufs = [torch.empty(n + 2 * GUARD, device="cuda") for _ in range(4)]
    alpha = 1e-3
    rng = np.random.default_rng(5)
    stripes = [np.arange(c - (1 << 16), c + (1 << 16)) for c in ((1 << 29), (1 << 30), TWO31)] + [np.arange(n - (1 << 20), n)]
    idx = np.unique(np.concatenate(stripes + [rng.integers(0, n, 1 << 20)]))
    gi = torch.as_tensor(idx + GUARD, device="cuda")
    weights = torch.arange(C, device="cuda", dtype=torch.int64) * 2 * 0x9E3779B97F4A7C1 + 1
    digests = {}
    try:
        for cap in (0, 1):
            _adam_fill(bufs, n, 17)
            before = [t[gi].clone() for t in bufs]
            udh.lib.check(udh.L.udh_set_adam_grid(cap), "udh_set_adam_grid")
            ts = time.time()
            udh.lib.check(udh.L.udh_adam_step(*(P_(t[GUARD:]) for t in bufs), n, alpha, 0.9, 0.999, 1e-8, 1.0, 1, None), "udh_adam_step")
            torch.cuda.synchronize()
            dt = time.time() - ts
            p, g, m, v = bufs
            for t, name in zip(bufs, "pgmv"):
                assert (t[:GUARD] == SENTINEL).all() and (t[GUARD + n:] == SENTINEL).all(), "cap %d: guard band of %s written" % (cap, name)
            assert not g[GUARD:GUARD + n].any(), "cap %d: the gradient was not zeroed" % cap
            P64, M64, V64 = OPT.adam64(*before, alpha)
            ep, em, ev = OPT.adam_bound(*before, alpha)
            worst = {}
            for name, got, ref, bound in (("p", p[gi], P64, ep), ("m", m[gi], M64, em), ("v", v[gi], V64, ev)):
                d = (got.double() - ref).abs()
                bad = (d > bound).nonzero().flatten()
                assert bad.numel() == 0, "cap %d: %s' off the Adam bound at %d elements, first at flat index %d: %.3e > %.3e" % (
                    cap, name, bad.numel(), int(idx[bad[0].item()]), d[bad[0]].item(), bound[bad[0]].item())
                hi = torch.as_tensor(idx >= TWO31, device="cuda")
                worst[name] = ((d / bound).max().item(), (d[hi] / bound[hi]).max().item())
            digests[cap] = [_digest(t, n, weights) for t in (p, m, v)]
            print("Adam n=%d grid cap %d: %.1f ms; %d elements checked (stripes at 2^29, 2^30, 2^31 floats, the last 2^20, 2^20 random): "
                  "p' %.3f (past 2^31: %.3f), m' %.3f (%.3f), v' %.3f (%.3f) of the bound; guard bands intact"
                  % (n, cap, dt * 1e3, idx.size, *worst["p"], *worst["m"], *worst["v"]))
    finally:
        udh.L.udh_set_adam_grid(0)
        release(*bufs)
    for name, a, b in zip("pmv", digests[0], digests[1]):
        diff = [i for i, (u, w) in enumerate(zip(a, b)) if u != w]
        assert not diff, "%s': grid caps 0 and 1 differ in chunks %s (of %d floats)" % (name, diff[:8], C)
    print("Adam: grid caps 0 and 1 bit-identical over all %d floats (%.1f s)" % (n, time.time() - t0))


# ------------------------------------------------------------------------------------------------ 4. the engine at large P
ENGINE_CASES = [(1, 384), (2, 384), (1, 1408)]


def engine_need(udh, B, Pz):
    n = udh.L.udh_param_total_floats(Pz)
    return 4 * 4 * n, udh.L.udh_cnn_workspace_bytes(B, Pz, udh.lib.NUMERIC_FP32)


def _conv64_full(x, w, bias, dgrad):
    """ref_conv of the whole tensor, assembled from row bands (bounded temporaries)."""
    B, H, W_ = x.shape[:3]
    C = w.shape[2] if dgrad else w.shape[3]
    out = torch.empty(B, H, W_, C, dtype=torch.float64, device=x.device)
    step = band_rows(x, max(C, x.shape[3]))
    for y0 in range(0, H, step):
        out[:, y0:y0 + step] = ref_conv_rows(x, w, bias, dgrad, y0, min(H, y0 + step))
    return out


def fp64_forward(eng, I1, I2, m1, m2):
    """pred_h4p of the engine's parameters in float64 on the device (fc1 in row chunks), with its dropout masks."""
    p = eng.named_parameters()
    names = list(p)
    x = torch.cat([I1, I2], dim=3)
    for i in range(8):
        w, b = p[names[2 * i]], p[names[2 * i + 1]]
        x = F.relu(_conv64_full(x, w, b, False))
        if i in (1, 3, 5):
            x = S.pool_fwd(x)
    a = (x * m1.double() * 2).reshape(eng.B, -1)
    W1 = p[names[16]]
    y = torch.zeros(eng.B, 1024, dtype=torch.float64, device="cuda")
    for r0 in range(0, W1.shape[0], ROWS):
        y += a[:, r0:r0 + ROWS] @ W1[r0:r0 + ROWS].double()
    fc1 = F.relu(y + p[names[17]].double()) * m2.double() * 2
    return fc1 @ p[names[18]].double() + p[names[19]].double()


def _engine(udh, B, Pz, seed, **kw):
    h, w = image_size(Pz)
    eng = udh.engine.HomographyEngine(B, patch_size=Pz, img_h=h, img_w=w, numeric="fp32", seed=None, **kw)
    eng.load_flat(udh.params.init_flat_large(seed, Pz))
    return eng


@pytest.mark.parametrize("BP", ENGINE_CASES, ids=_ids)
def test_engine_large_patch(udh, BP):
    """The engine at a large patch on init_flat_large weights and images with flat regions:
    (a) every conv activation within gamma_{K+1} of float64 on the engine's own input activation (row bands), every pool
        bit-identical to the rule on its pre-pool activation;
    (b) udh_cnn_bwd (train mode, a chosen dh4p) against a float64 backward on its own gates: relative L2 per tensor within
        the 5e-6 of test_gpu_fp32_certify.py, fc1's weight gradient summed in row chunks;
    (c) one h_loss step (forward, backward, Adam): pred_h4p within 1e-5 relative of a float64 forward with the engine's
        dropout masks, and Adam's update of 2^16 sampled fc1 weights (past flat index 2^31 where the buffer reaches it) within
        oracle.optim.adam_bound of the float64 update from the step's own gradient."""
    B, Pz = BP
    nparam, ws = engine_need(udh, B, Pz)
    need_device(nparam + ws + 8 * 4 * (Pz ** 2) * 64 * B + 8 * 4 * ROWS * 1024, "engine B=%d P=%d" % (B, Pz))
    need_host(nparam // 4 + 8 * (1 << 24) + 4 * GiB, "engine B=%d P=%d" % (B, Pz))
    t0 = time.time()
    eng = _engine(udh, B, Pz, 3, loss_type="h_loss", lr=5e-4)
    try:
        _engine_case(udh, eng, t0)
    finally:
        release_engine(eng)


def _engine_case(udh, eng, t0):
    B, Pz = eng.B, eng.Pz
    batch = flat_batch(3, B, Pz)
    db = {k: (v.cuda().contiguous() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}
    I1, I2 = db["I1_aug"], db["I2_aug"]
    # (a) forward layer by layer
    cnn_fwd(udh, eng, I1, I2, False, 0)
    A = acts(eng)
    report = []
    for i in range(8):
        w, b = conv_params(eng, i)
        frac = check_conv_banded(A[i], layer_input(A, I1, I2, i), w, b, False, "engine B=%d P=%d layer %d" % (B, Pz, i), relu=True)
        report.append("conv%d %.3f" % (i, frac))
    gen = torch.Generator(device="cuda").manual_seed(B + Pz)
    for pi, src in ((8, 1), (9, 3), (10, 5)):
        check_exact(A[pi], S.pool_fwd(A[src]).double(), "engine B=%d P=%d pool%d" % (B, Pz, pi - 7))
        dout = torch.randn(A[pi].shape, device="cuda", generator=gen)
        ties, zeros = check_pool(udh, A[src].contiguous(), dout, "engine B=%d P=%d pool%d" % (B, Pz, pi - 7))
        del dout
        assert ties > 0 and zeros > 0, (pi, ties, zeros)
        report.append("pool%d exact (%d ties, %d zero windows)" % (pi - 7, ties, zeros))
    print("engine forward B=%d P=%d, fraction of the float64 bound: %s (%.1f s)" % (B, Pz, ", ".join(report), time.time() - t0))
    # (b) backward on its own gates
    cnn_fwd(udh, eng, I1, I2, True, 0xC0FFEE + B)
    A = acts(eng)
    dh4p = torch.randn(B, 8, device="cuda", generator=torch.Generator(device="cuda").manual_seed(B)).contiguous()
    eng.grads.zero_()
    udh.lib.check(udh.L.udh_cnn_bwd(P_(eng.params), P_(I1), P_(I2), P_(dh4p), P_(eng.grads), P_(eng.ws), eng.ws_bytes, B, Pz, 1,
                                    udh.lib.NUMERIC_FP32, None), "udh_cnn_bwd")
    torch.cuda.synchronize()
    errs = fp64_backward_rel_l2(eng, A, I1, I2, dh4p.double())
    worst = max(errs.values())
    print("engine backward B=%d P=%d vs float64 on its own gates (bound 5e-6), worst %.3e (%s): %s (%.1f s)"
          % (B, Pz, worst, max(errs, key=errs.get), ", ".join("%s %.1e" % (k.split("/", 1)[1], v) for k, v in errs.items()),
             time.time() - t0))
    assert worst <= 5e-6, errs
    del A
    # (c) one h_loss step
    eng.grads.zero_()
    out = eng.forward(db, train=True)
    m1, m2 = eng.dropout_masks()
    pred64 = fp64_forward(eng, I1.double(), I2.double(), m1.reshape(B, Pz // 8, Pz // 8, 128), m2)
    scale = pred64.abs().max().item()
    e = ((out["pred_h4p"].double() - pred64).abs().max() / scale).item()
    eng.backward(db, out)
    s = eng.specs["model/fc1/fc1/weights"]
    rng = np.random.default_rng(B + Pz)
    lo = max(s.offset, TWO31) if s.offset + s.size > TWO31 else s.offset
    sample = torch.as_tensor(np.unique(np.concatenate([rng.integers(lo, s.offset + s.size, 1 << 16),
                                                       np.arange(s.offset + s.size - 64, s.offset + s.size)])), device="cuda")
    before = [t[sample].clone() for t in (eng.params, eng.grads, eng.adam_m, eng.adam_v)]
    alpha = eng._alpha()[1]
    eng.update()
    torch.cuda.synchronize()
    P64 = OPT.adam64(*before, alpha)[0]
    ep = OPT.adam_bound(*before, alpha)[0]
    d = (eng.params[sample].double() - P64).abs()
    moved, live = int((eng.params[sample] != before[0]).sum()), int((before[1] != 0).sum())
    print("engine step B=%d P=%d: pred_h4p rel err %.2e vs float64 (max |pred_h4p| %.1f px, bound 1e-5); Adam on %d fc1 weights "
          "from flat index %d (%s 2^31): %.3f of the bound, %d with a nonzero gradient, %d moved (%.1f s)"
          % (B, Pz, e, scale, sample.numel(), lo, ">=" if lo >= TWO31 else "<", (d / ep).max().item(), live, moved, time.time() - t0))
    assert scale > 10.0 and e <= 1e-5, (scale, e)
    assert (d <= ep).all(), "Adam's update of fc1 weights off the bound at %d of %d sampled elements" % (int((d > ep).sum()), sample.numel())
    assert live > 0 and moved >= live // 2, (live, moved)      # the weights with a gradient move (the rest keep m = 0)


def fp64_backward_rel_l2(eng, A, I1, I2, dh4p):
    """Relative L2 of each parameter gradient of the engine against the float64 backward on its own gates (ReLU masks from its
    activations, pool routing by the rule, its dropout masks), with fc1's weight gradient compared in row chunks and each
    conv's tensors formed one layer at a time."""
    p = eng.named_parameters()
    gr = eng.named_gradients()
    names = list(p)
    B = eng.B
    m1, m2 = (m.double() for m in eng.dropout_masks())
    rel = lambda got, ref: ((got.double() - ref).norm() / ref.norm().clamp_min(1e-300)).item()
    errs = {}
    a11 = A[11].double()
    fc1d = a11 * m2 * 2
    errs[names[18]] = rel(gr[names[18]], fc1d.t() @ dh4p)
    errs[names[19]] = rel(gr[names[19]], dh4p.sum(0))
    dfc1 = (dh4p @ p[names[18]].double().t()) * m2 * 2 * (a11 > 0)
    errs[names[17]] = rel(gr[names[17]], dfc1.sum(0))
    a4d = (A[7].double() * m1.reshape(A[7].shape) * 2).reshape(B, -1)
    W1, G1 = p[names[16]], gr[names[16]]
    num = den = 0.0
    g = torch.empty(B, W1.shape[0], dtype=torch.float64, device="cuda")
    for r0 in range(0, W1.shape[0], ROWS):
        r1 = min(W1.shape[0], r0 + ROWS)
        ref = a4d[:, r0:r1].t() @ dfc1
        num += (G1[r0:r1].double() - ref).square().sum().item()
        den += ref.square().sum().item()
        g[:, r0:r1] = dfc1 @ W1[r0:r1].double().t()
    errs[names[16]] = (num / max(den, 1e-300)) ** 0.5
    del a4d
    g = g.reshape(A[7].shape) * m1.reshape(A[7].shape) * 2 * (A[7] > 0)
    for i in range(7, -1, -1):
        x = layer_input(A, I1, I2, i)
        dW, dbias = ref_wgrad_banded(x, g)
        errs[names[2 * i]], errs[names[2 * i + 1]] = rel(gr[names[2 * i]], dW), rel(gr[names[2 * i + 1]], dbias)
        if i == 0:
            break
        d = _conv64_full(g, p[names[2 * i]], None, True)
        g = S.pool_bwd(A[i - 1].double(), d) if i in (2, 4, 6) else d * (A[i - 1] > 0)
        del d
    return errs


# ------------------------------------------------------------------------------------------------ 5. the checkpoint at P = 1152
def test_checkpoint_round_trip_P1152(udh):
    """save_tf_checkpoint(with_optimizer=False) of a P = 1152 engine (fc1: 2.72e9 floats, 10.9 GB, past every 32-bit size,
    offset and CRC length of the writer, the reader and udh_crc32c) loads into a fresh engine bit for bit; so does a .pt
    state_dict (parameters and both Adam moments) through torch.save / torch.load."""
    Pz, B = 1152, 1
    nparam, ws = engine_need(udh, B, Pz)
    n = nparam // 16
    # one engine at a time (params, grads, m, v and its workspace), the reference copy of the parameters, and one chunk of
    # regenerated moments plus its comparison mask; m and v are regenerated from their seed rather than copied
    need_device(nparam + ws + 4 * n + 5 * CHUNK, "checkpoint P=%d" % Pz)
    need_host(3 * 4 * n + 4 * GiB, "checkpoint P=%d" % Pz)
    tmp = tempfile.mkdtemp(prefix="udh_ckpt_")
    held = []
    try:
        disk = shutil.disk_usage(tmp).free
        if disk < 4 * 4 * n + GiB:          # the TF bundle (parameters) and the .pt file (parameters, m, v) side by side
            pytest.skip("checkpoint P=%d needs %.1f GiB of disk, %.1f GiB free" % (Pz, 4 * 4 * n / GiB, disk / GiB))
        print("checkpoint P=%d: %.1f GiB of disk free" % (Pz, disk / GiB))
        t0 = time.time()
        eng = _engine(udh, B, Pz, 4)
        held.append(eng)
        gen = torch.Generator(device="cuda").manual_seed(4)
        _fill_chunks(eng.adam_m, lambda t: t.normal_(generator=gen))
        _fill_chunks(eng.adam_v, lambda t: t.uniform_(generator=gen))
        eng.global_step = 77
        ref = eng.params.clone()
        held.append(ref)
        prefix = os.path.join(tmp, "model.ckpt-77")
        eng.save_tf_checkpoint(prefix, with_optimizer=False)
        size = os.path.getsize(prefix + ".data-00000-of-00001")
        assert size == 4 * sum(s.size for s in eng.specs.values()) + 4, size         # the tensors and the int32 step
        t_save = time.time() - t0
        sd_path = os.path.join(tmp, "state.pt")
        torch.save(eng.state_dict(), sd_path)
        release_engine(eng)
        del eng, held[0]
        torch.cuda.empty_cache()
        e2 = udh.engine.HomographyEngine(B, patch_size=Pz, img_h=image_size(Pz)[0], img_w=image_size(Pz)[1], numeric="fp32", seed=None)
        held.append(e2)
        t1 = time.time()
        e2.load_tf_checkpoint(prefix)
        t_load = time.time() - t1
        assert e2.global_step == 77
        assert_same_bits(e2.params, lambda a, b: ref[a:b], "the TF checkpoint's parameters")
        assert not e2.adam_m.any() and not e2.adam_v.any()
        os.remove(prefix + ".data-00000-of-00001")
        e2.params.zero_()
        e2.load_state_dict(torch.load(sd_path, mmap=True))
        assert_same_bits(e2.params, lambda a, b: ref[a:b], "the .pt state_dict's parameters")
        gen = torch.Generator(device="cuda").manual_seed(4)              # the moments again, chunk by chunk, from their seed
        assert_same_bits(e2.adam_m, lambda a, b: torch.empty(b - a, device="cuda").normal_(generator=gen), "the .pt state_dict's adam_m")
        assert_same_bits(e2.adam_v, lambda a, b: torch.empty(b - a, device="cuda").uniform_(generator=gen), "the .pt state_dict's adam_v")
        assert e2.global_step == 77
        print("checkpoint P=%d: %d parameters (fc1 %d floats, %.1f GB); TF bundle %.1f GB written in %.1f s, read back in %.1f s, "
              "bit-identical; .pt state_dict bit-identical (%.1f s in all)"
              % (Pz, n, e2.specs["model/fc1/fc1/weights"].size, 4e-9 * e2.specs["model/fc1/fc1/weights"].size, size / 1e9, t_save,
                 t_load, time.time() - t0))
    finally:
        for h in held:
            if isinstance(h, torch.Tensor):
                release(h)
            else:
                release_engine(h)
        shutil.rmtree(tmp, ignore_errors=True)

