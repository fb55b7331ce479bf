"""Helpers of the fp32 CUDA-core engine's certification (UDH_NUMERIC_FP32, csrc/cnn_simt.cu), shared by
test_gpu_fp32_certify.py (P = 128, 256) and test_gpu_fp32_large_patch.py (P up to 1408): the layer kernels through the C ABI,
their float64 references (whole tensors, or row bands with their halo so that a 1408-pixel layer stays in bounded memory),
the exact / restated / bounded checks, and the engine's activations and batches."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import oracle as O
from oracle import simt_fp32 as S

P_ = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None

# conv instances of the step: (name, P / spatial size, cin, cout); conv2_1 / conv2_2 share one, and so do conv4_1 / conv4_2
CONVS = [("conv1_1", 1, 2, 64), ("conv1_2", 1, 64, 64), ("conv2_x", 2, 64, 64), ("conv3_1", 4, 64, 128),
         ("conv3_2", 4, 128, 128), ("conv4_x", 8, 128, 128)]
# dgrad instances: the layer's shape and whether the step fuses the ReLU mask of the layer below (not when a pool is below)
DGRADS = [("conv1_2", 1, 64, 64, True), ("conv2_1", 2, 64, 64, False), ("conv2_2", 2, 64, 64, True), ("conv3_1", 4, 64, 128, False),
          ("conv3_2", 4, 128, 128, True), ("conv4_1", 8, 128, 128, False), ("conv4_2", 8, 128, 128, True)]
POOLS = [("pool1", 1, 64), ("pool2", 2, 64), ("pool3", 4, 128)]              # (name, P / pre-pool size, channels)
FULL_IMAGE_STEPS = 4e7           # restate every output of the first and last image when that is <= this many fmaf steps
BAND_ELEMS = 1 << 25             # float64 elements of one row band of a reference (256 MB)


# ------------------------------------------------------------------------------------------------ kernels through the C ABI
def simt_conv(udh, x, w, bias=None, mask=None, relu=0, dgrad=0, x2=None):
    B, H, W = x.shape[:3]
    cin, cout = w.shape[2], w.shape[3]
    out = torch.full((B, H, W, cin if dgrad else cout), float("nan"), device="cuda")
    wrot = torch.empty(9 * cin * cout, device="cuda") if dgrad else None
    rc = udh.L.udh_debug_simt_conv(P_(x), P_(x2), P_(w), P_(bias), P_(mask), P_(out), P_(wrot), B, H, W, cin, cout, relu, dgrad, None)
    assert rc == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    return out


def simt_wgrad(udh, x, g, cin, x2=None):
    B, H, W, cout = g.shape
    dW = torch.zeros(3, 3, cin, cout, device="cuda"); db = torch.zeros(cout, device="cuda")
    part = [ctypes.c_int() for _ in range(3)]
    rc = udh.L.udh_debug_simt_wgrad(P_(x), P_(x2), P_(g), P_(dW), P_(db), B, H, W, cin, cout, *[ctypes.byref(v) for v in part], None)
    assert rc == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    return dW, db, tuple(v.value for v in part)


def simt_pool(udh, x, dout=None):
    B, H, W, C = x.shape
    out = torch.full((B, H // 2, W // 2, C), float("nan"), device="cuda")
    din = torch.full_like(x, float("nan")) if dout is not None else None
    assert udh.L.udh_debug_simt_pool(P_(x), P_(out), P_(dout), P_(din), B, H, W, C, None) == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    return out, din


# ------------------------------------------------------------------------------------------------ float64 references
def _kernel64(w, dgrad):
    wk = torch.flip(w, dims=(0, 1)).permute(2, 3, 0, 1) if dgrad else w.permute(3, 2, 0, 1)
    return wk.double().contiguous()


def ref_conv(x, w, bias=None, dgrad=False):
    """float64 conv3x3 (pad 1) + bias of NHWC x; dgrad: the gradient w.r.t. the layer's input of g = x."""
    r = F.conv2d(x.double().permute(0, 3, 1, 2), _kernel64(w, dgrad), None if bias is None else bias.double(), padding=1)
    return r.permute(0, 2, 3, 1)


def _rows_with_halo(x, y0, y1):
    """float64 rows [y0 - 1, y1 + 1) of NHWC x, zero rows outside the image: the input of output rows [y0, y1)."""
    H = x.shape[1]
    lo, hi = max(y0 - 1, 0), min(y1 + 1, H)
    return F.pad(x[:, lo:hi].double(), (0, 0, 0, 0, lo - (y0 - 1), (y1 + 1) - hi))


def ref_conv_rows(x, w, bias, dgrad, y0, y1, absolute=False):
    """Output rows [y0, y1) of ref_conv (of the |x| |w| |b| conv with absolute=True)."""
    xs, wk = _rows_with_halo(x, y0, y1), _kernel64(w, dgrad)
    b = None if bias is None else bias.double()
    if absolute:
        xs, wk, b = xs.abs(), wk.abs(), None if b is None else b.abs()
    return F.conv2d(xs.permute(0, 3, 1, 2), wk, b, padding=(0, 1)).permute(0, 2, 3, 1)


def ref_wgrad(x, g):
    dW = torch.nn.grad.conv2d_weight(x.double().permute(0, 3, 1, 2), (g.shape[3], x.shape[3], 3, 3), g.double().permute(0, 3, 1, 2),
                                     padding=1)
    return dW.permute(2, 3, 1, 0), g.double().sum(dim=(0, 1, 2))


def band_rows(x, channels):
    """Rows per band so that one float64 band of [B, rows, W, channels] holds about BAND_ELEMS elements."""
    return max(1, min(x.shape[1], BAND_ELEMS // (x.shape[0] * x.shape[2] * channels)))


def ref_wgrad_banded(x, g, absolute=False):
    """ref_wgrad summed over row bands of the output (each band with its input halo): (dW, db) in float64, or the sums of
    |x| |g| and |g| with absolute=True."""
    B, H, W, cout = g.shape
    cin = x.shape[3]
    dW = torch.zeros(cout, cin, 3, 3, dtype=torch.float64, device=g.device)
    db = torch.zeros(cout, dtype=torch.float64, device=g.device)
    step = band_rows(x, max(cin, cout))
    for y0 in range(0, H, step):
        y1 = min(H, y0 + step)
        xs, gs = _rows_with_halo(x, y0, y1), g[:, y0:y1].double()
        if absolute:
            xs, gs = xs.abs(), gs.abs()
        dW += torch.nn.grad.conv2d_weight(xs.permute(0, 3, 1, 2), (cout, cin, 3, 3), gs.permute(0, 3, 1, 2), padding=(0, 1))
        db += gs.sum(dim=(0, 1, 2))
    return dW.permute(2, 3, 1, 0), db


def conv_bound(x, w, bias, dgrad):
    kin = w.shape[3] if dgrad else w.shape[2]
    return float(S.gamma(9 * kin + 1)) * ref_conv(x.abs(), w.abs(), None if bias is None else bias.abs(), dgrad)


def _pos(shape, flat_idx):
    return tuple(int(v) for v in np.unravel_index(int(flat_idx), tuple(shape)))


def _at(shape, flat_idx, off):
    return tuple(v + o for v, o in zip(_pos(shape, flat_idx), off or (0,) * len(shape)))


def check_exact(got, ref, what, names="n,y,x,c", off=None):
    """got equals the float64 ref on every element.  off: per-dimension offset of this slice in the whole tensor (a row band,
    a chunk of rows), added to the positions the message names."""
    bad = (got.double() != ref)
    if bad.any():
        idx = bad.flatten().nonzero().flatten()[:4].tolist()
        at = "; ".join("(%s)=%s: %r vs %r" % (names, _at(ref.shape, i, off), got.flatten()[i].item(), ref.flatten()[i].item()) for i in idx)
        pytest.fail("%s: %d elements differ from float64 with exact operands: %s" % (what, int(bad.sum()), at))


def check_bound(got, ref, bound, what, names="n,y,x,c", off=None):
    """Every element within its bound; returns the largest fraction of the bound reached.  The message names the image and
    position of the worst offenders (off as in check_exact)."""
    d = (got.double() - ref).abs()
    bad = d > bound
    if bad.any():
        frac = torch.where(bad, d / bound.clamp_min(1e-300), torch.zeros_like(d)).flatten()
        idx = frac.topk(min(4, int(bad.sum()))).indices.tolist()
        at = "; ".join("(%s)=%s: err %.3e > bound %.3e" % (names, _at(ref.shape, i, off), d.flatten()[i].item(), bound.flatten()[i].item())
                       for i in idx)
        pytest.fail("%s: %d elements over the float64 bound: %s" % (what, int(bad.sum()), at))
    pos = bound > 0
    return (d[pos] / bound[pos]).max().item() if pos.any() else 0.0


def check_conv_banded(got, x, w, bias, dgrad, what, relu=False, mask=None, exact=False):
    """got (a conv / dgrad output) against its float64 reference, one row band at a time: bit-equal with exact=True (exact
    operands), else every element within gamma_{K+1} (|x| |w| + |b|).  relu / mask: the output's ReLU and fused mask
    (mask <= 0 forces 0, and there the bound is 0).  Returns the largest fraction of the bound reached."""
    B, H, W, C = got.shape
    kin = w.shape[3] if dgrad else w.shape[2]
    g_ = float(S.gamma(9 * kin + 1))
    worst, step = 0.0, band_rows(x, max(C, x.shape[3]))
    for y0 in range(0, H, step):
        y1 = min(H, y0 + step)
        ref = ref_conv_rows(x, w, bias, dgrad, y0, y1)
        if relu:
            ref = F.relu(ref)
        keep = None if mask is None else (mask[:, y0:y1] > 0)
        if keep is not None:
            ref = ref * keep
        if exact:
            check_exact(got[:, y0:y1], ref, what, off=(0, y0, 0, 0))
            continue
        bound = g_ * ref_conv_rows(x, w, bias, dgrad, y0, y1, absolute=True)
        if keep is not None:
            bound = bound * keep
        worst = max(worst, check_bound(got[:, y0:y1], ref, bound, what, off=(0, y0, 0, 0)))
    return worst


def int_tensor(g, shape, lo=-2, hi=2):
    return torch.randint(lo, hi + 1, shape, device="cuda", generator=g).float().contiguous()


# ------------------------------------------------------------------------------------------------ restated chains
def chain_sample(B, H, W, C, K, seed):
    """Output elements whose chains are restated: every output of the first and last image when that is cheap, otherwise
    the top-left 8x16 tile of the first image and the bottom-right one of the last at 16 channels (every CTA channel group
    of four is hit at 64 channels), plus 2048 random elements."""
    last = B - 1
    if 2 * H * W * C * K <= FULL_IMAGE_STEPS:
        n, y, x, c = (a.reshape(-1) for a in np.meshgrid(np.array(sorted({0, last})), np.arange(H), np.arange(W), np.arange(C),
                                                          indexing="ij"))
    else:
        ch = np.linspace(0, C - 1, 16).round().astype(int)
        parts = []
        for nn, y0, x0 in ((0, 0, 0), (last, H - 8, W - 16)):
            yy, xx, cc = (a.reshape(-1) for a in np.meshgrid(np.arange(y0, y0 + 8), np.arange(x0, x0 + 16), ch, indexing="ij"))
            parts.append((np.full_like(yy, nn), yy, xx, cc))
        n, y, x, c = (np.concatenate(v) for v in zip(*parts))
    rng = np.random.default_rng(seed)
    m = 2048
    return (np.concatenate([n, rng.integers(0, B, m)]), np.concatenate([y, rng.integers(0, H, m)]),
            np.concatenate([x, rng.integers(0, W, m)]), np.concatenate([c, rng.integers(0, C, m)]))


def check_chain(got, x, w, bias, mask, relu, dgrad, seed, what, x2=None):
    B, H, W, C = got.shape
    kin = w.shape[3] if dgrad else w.shape[2]
    n, y, xx, c = chain_sample(B, H, W, C, 9 * kin, seed)
    want = S.conv_chain(x, w, n, y, xx, c, bias=bias, relu=relu, mask=mask, dgrad=dgrad, x2=x2)
    have = got[torch.as_tensor(n), torch.as_tensor(y), torch.as_tensor(xx), torch.as_tensor(c)].cpu().numpy()
    bad = np.nonzero(have != want)[0]
    assert bad.size == 0, "%s: %d of %d restated elements differ, e.g. %s" % (
        what, bad.size, len(n), "; ".join("(n,y,x,c)=(%d,%d,%d,%d): %r vs restated %r" % (n[i], y[i], xx[i], c[i], have[i], want[i])
                                         for i in bad[:4]))
    return len(n)


def check_partials(dW, db, x, g, part, E, seed, what, x2=None):
    """dW / db of E sampled elements within gamma_{m-1} sum|p| of the float64 sum of their restated thread partials."""
    cin, cout = dW.shape[2], dW.shape[3]
    rng = np.random.default_rng(seed)
    ky, kx, ci, co = rng.integers(0, 3, E), rng.integers(0, 3, E), rng.integers(0, cin, E), rng.integers(0, cout, E)
    worst = 0.0
    for name, p, got in (("dW", S.wgrad_partials(x, g, part, ky, kx, ci, co, x2=x2), dW[ky, kx, ci, co]),
                         ("db", S.bias_partials(g, part, co), db[co])):
        s, bound = S.sum_bound(p)
        d = np.abs(got.double().cpu().numpy() - s)
        bad = np.nonzero(d > bound)[0]
        assert bad.size == 0, "%s %s: partition %s, %s" % (what, name, part, "; ".join(
            "(ky,kx,ci,co)=(%d,%d,%d,%d): |dW - sum p| %.3e > %.3e" % (ky[i], kx[i], ci[i], co[i], d[i], bound[i]) for i in bad[:4]))
        worst = max(worst, float((d / np.maximum(bound, 1e-300)).max()))
    return worst


# ------------------------------------------------------------------------------------------------ pools
def check_pool(udh, x, dout, what):
    out, din = simt_pool(udh, x, dout)
    check_exact(out, S.pool_fwd(x).double(), what + " forward")          # values; the sign of a zero maximum is not pinned
    want = S.pool_bwd(x, dout)
    bad = din.view(torch.int32) != want.view(torch.int32)
    assert not bad.any(), "%s backward: %d elements differ from the routing rule, first at (n,y,x,c)=%s" % (
        what, int(bad.sum()), _pos(x.shape, bad.flatten().nonzero()[0].item()))
    a, b, c, d = S._windows(x)
    m = S.pool_fwd(x)
    ties = ((a == m).int() + (b == m).int() + (c == m).int() + (d == m).int() >= 2) & (m > 0)
    return int(ties.sum()), int((m == 0).sum())


# ------------------------------------------------------------------------------------------------ the engine
def image_size(Pz):
    """(img_h, img_w) of the synthetic images a Pz patch is cut from: 240 x 320 at the reference's 128, 360 x 480 at 256,
    and the patch plus the same margins (rho = 45 on each side, and more across) above that."""
    return {128: (240, 320), 256: (360, 480)}.get(Pz, (Pz + 104, Pz + 224))


def flat_batch(seed, B, Pz):
    """A seeded batch whose patches have flat (saturated) regions: exact ties in every pool and zero-gradient plateaus."""
    h, w = image_size(Pz)
    batch = O.make_batch(seed, B, img_h=h, img_w=w, patch=Pz)
    for k in ("I1_aug", "I2_aug"):
        t = batch[k].clone()
        t[:, Pz // 8: Pz // 2, Pz // 4: 3 * Pz // 4] = 1.5
        t[:, 5 * Pz // 8:, : Pz // 3] = -1.25
        batch[k] = t
    return batch


def cnn_fwd(udh, eng, I1, I2, train, seed):
    h4p = torch.empty(eng.B, 8, device="cuda")
    udh.lib.check(udh.L.udh_cnn_fwd(P_(eng.params), P_(I1), P_(I2), P_(h4p), P_(eng.ws), eng.ws_bytes, eng.B, eng.Pz, int(train), seed,
                                    udh.lib.NUMERIC_FP32, None), "udh_cnn_fwd")
    torch.cuda.synchronize()
    return h4p


def acts(eng):
    B, Pz = eng.B, eng.Pz
    shape = {i: (B, Pz // d, Pz // d, c) for i, (_, d, _, c) in enumerate([CONVS[0], CONVS[1], CONVS[2], CONVS[2], CONVS[3], CONVS[4],
                                                                         CONVS[5], CONVS[5]])}
    shape.update({8: (B, Pz // 2, Pz // 2, 64), 9: (B, Pz // 4, Pz // 4, 64), 10: (B, Pz // 8, Pz // 8, 128), 11: (B, 1024)})
    return {i: eng.activation(i).reshape(s) for i, s in shape.items()}


def layer_input(acts, I1, I2, i):
    if i == 0:
        return torch.cat([I1, I2], dim=3)
    return acts[8 + (i - 2) // 2] if i in (2, 4, 6) else acts[i - 1]


def conv_params(eng, i, dtype=None):
    p = eng.named_parameters()
    names = list(p)
    w, b = p[names[2 * i]], p[names[2 * i + 1]]
    return (w, b) if dtype is None else (w.to(dtype), b.to(dtype))
