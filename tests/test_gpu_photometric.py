"""The photometric path against fp64 on the kernels' own gates (-m gpu): warp backward for every loss type, warp forward
pixels, the six sums and their finalisation, SSIM forward / backward, the bit-exact resamplers, the DLT and udh_h4p_loss.

oracle/warp_fp32.py restates every fp32 gate of csrc/warp.cu (coordinates, clipped cells, weights, gray values, the L1
sign and the L1-smooth clamp) bit for bit.  With the gates identical, what separates a kernel from the fp64 evaluation
on those gates is the kernel's own fp32 rounding, and each bound below is derived from that rounding rather than from
the ~1e-2 flip noise that a comparison with the fp64 oracle's own coordinates has to absorb (tests/test_gpu_parity.py).
Every check prints its worst measured value next to its bound.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import warp_fp32 as R

pytestmark = pytest.mark.gpu

f32 = np.float32
U = R.U32
IMG_H, IMG_W = 240, 320


@pytest.fixture(scope="module")
def udh():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from unsuperviseddeephomographyral2018_b200 import _lib, ops, synthetic
    _lib.require_device()

    class NS:
        pass
    ns = NS()
    ns.lib, ns.ops, ns.synthetic = _lib, ops, synthetic
    return ns


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _report(what, worst, bound):
    print("  %-58s worst %.3e   bound %.3e" % (what, worst, bound))


# ------------------------------------------------------------------------------------------------ inputs
def _homographies(kind, B, ox, oy, pts_w, rng):
    """[B,9] fp32 pixel-unit H.  'mix' cycles through gt + noise, a strongly projective H whose horizon (t_s = 0) crosses
    the window, an integer translation and the identity."""
    H = np.zeros((B, 9))
    for b in range(B):
        k = b % 4 if kind == "mix" else 0
        if k == 0:
            x0, y0 = float(ox[b]), float(oy[b])
            p1 = np.array([x0, y0, x0 + pts_w, y0, x0 + pts_w, y0 + pts_w, x0, y0 + pts_w])
            p2 = p1 + rng.integers(-45, 46, 8) + rng.normal(0, 2.0, 8)
            A, rhs = R.dlt_system(p1[None].astype(f32), (p2 - p1)[None].astype(f32))
            H[b, :8] = np.linalg.solve(A[0], rhs[0]); H[b, 8] = 1
        elif k == 1:
            H[b] = [1.0, 0.05, 3.0, -0.02, 1.0, -2.0, -1.0 / (ox[b] + 64.3 + 0.01 * b), 1e-4, 1.0]
        elif k == 2:
            H[b] = [1, 0, rng.integers(-20, 21), 0, 1, rng.integers(-20, 21), 0, 0, 1]
        else:
            H[b] = [1, 0, 0, 0, 1, 0, 0, 0, 1]
    return torch.tensor(H.astype(f32)).cuda()


class Case:
    pass


def _sel(B):
    """Samples restated pixel by pixel: the first and last eight and four in the middle, i.e. every H kind of the 'mix'
    cycle several times and the batch's tail.  The kernels treat every sample alike (one CTA row per sample), so a spread
    of samples covers the indexing; the sums and the step's per-sample outputs are still checked for every sample."""
    if B <= 20:
        return np.arange(B)
    return np.unique(np.r_[0:8, B // 2 - 2:B // 2 + 2, B - 8:B])


def _inputs(udh, B, C, pw, ph, origins, idx_kind, seed):
    """Source image from the fast synthetic generator, windows at `origins` ('rand' = the generator's, 'extreme' = the four
    corner-most 128-windows, None = the full grid), I2 = the warp under a nearby H plus noise."""
    rng = np.random.default_rng(seed)
    fb = udh.synthetic.make_batch_fast(B, seed=seed, want_rgb=(C == 3))
    I = (fb["I_aug_rgb"] if C == 3 else fb["I_aug"]).contiguous()
    if origins is None:
        ox = oy = np.zeros(B, np.int64)
    elif origins == "extreme":
        corners = [(0, 0), (192, 0), (0, 112), (192, 112)]
        ox = np.array([corners[b % 4][0] for b in range(B)]); oy = np.array([corners[b % 4][1] for b in range(B)])
    else:
        p = fb["pts1"].cpu().numpy()
        ox, oy = p[:, 0].astype(np.int64), p[:, 1].astype(np.int64)
    if origins is None:
        idx = None
    elif idx_kind == "table":
        yy, xx = np.meshgrid(np.arange(ph), np.arange(pw), indexing="ij")
        idx = torch.tensor(((yy[None] + oy[:, None, None]) * IMG_W + xx[None] + ox[:, None, None]).reshape(B, -1).astype(np.int32)).cuda()
    else:
        idx = torch.tensor((oy * IMG_W + ox).astype(np.int32)).cuda()          # one origin per sample, stride 1
    H = _homographies("mix", B, ox, oy, 128, rng)
    H_near = (H.double() * (1 + 1e-3 * torch.tensor(rng.normal(size=(B, 9)), device="cuda"))).float()
    H_near[:, 8] = 1
    p_near, _ = udh.ops.warp_loss_forward(I, H_near.contiguous(), None, idx, pw, ph)
    I2 = (p_near[..., 0] + 0.1 * torch.tensor(rng.normal(size=(B, ph, pw)).astype(f32), device="cuda")).contiguous()
    I2[:, ::7, ::5] = p_near[:, ::7, ::5, 0]               # some pixels where pred may equal I2 exactly (d == 0)
    c = Case()
    c.B, c.C, c.pw, c.ph, c.I, c.H, c.I2, c.idx, c.ox, c.oy = B, C, pw, ph, I, H.contiguous(), I2, idx, ox, oy
    return c


def _make_case(udh, B, C, pw, ph, origins, idx_kind, seed):
    c = _inputs(udh, B, C, pw, ph, origins, idx_kind, seed)
    I, I2, idx, ox, oy = c.I, c.I2, c.idx, c.ox, c.oy
    c.sel = _sel(B)
    c.pred, c.sums = udh.ops.warp_loss_forward(I, c.H, I2, idx, pw, ph)
    torch.cuda.synchronize()
    c.I_cpu = I[torch.tensor(c.sel, device="cuda")].cpu().numpy()
    c.H_cpu = c.H.cpu().numpy()[c.sel]
    c.t = R.warp_window(c.I_cpu, c.H_cpu, ox[c.sel], oy[c.sel], pw, ph)
    c.pred_cpu = c.pred[..., 0].cpu().numpy()
    c.I2_cpu = I2.cpu().numpy()
    return c


CASES = {
    "win_B1_C1_table": (1, 1, 128, 128, "rand", "table"),
    "win_B128_C1_table": (128, 1, 128, 128, "rand", "table"),
    "win_B128_C3_origin": (128, 3, 128, 128, "rand", "origin"),
    "win_B129_C1_extreme_origin": (129, 1, 128, 128, "extreme", "origin"),
    "win_B129_C3_extreme_table": (129, 3, 128, 128, "extreme", "table"),
    "win_B1100_C1_origin": (1100, 1, 128, 128, "rand", "origin"),
    "win_B1100_C3_table": (1100, 3, 128, 128, "rand", "table"),
    "full_B1_C1": (1, 1, IMG_W, IMG_H, None, None),
    "full_B64_C1": (64, 1, IMG_W, IMG_H, None, None),
    "full_B1_C3": (1, 3, IMG_W, IMG_H, None, None),
    "full_B64_C3": (64, 3, IMG_W, IMG_H, None, None),
}
_cache = {}


@pytest.fixture(scope="module", params=list(CASES))
def case(request, udh):
    name = request.param
    if name not in _cache:
        _cache.clear()                                        # one case resident at a time
        _cache[name] = _make_case(udh, *CASES[name], seed=len(name) * 31 + CASES[name][0])
    c = _cache[name]
    c.name = name
    return c


# ------------------------------------------------------------------------------------------------ a. backward
def _bwd_reference(c, loss_type, L, sums, dpred_cpu):
    """fp64 dH' [S,9] and sum |term| [S,9] on the restated gates for the selected samples."""
    t = c.t
    n = float(c.B * c.pw * c.ph)
    pv = t["pv"].astype(np.float64)
    tg = c.I2_cpu[c.sel].astype(np.float64)
    d32 = (t["pv"] - c.I2_cpu[c.sel]).astype(f32)             # the kernel's fp32 d: its sign / clamp are the gates
    d = d32.astype(np.float64)
    if loss_type == L.LOSS_L1:
        gp = np.sign(d) / n; ga = np.full_like(gp, 1.0 / n)
    elif loss_type == L.LOSS_REC:
        k = 1.0 / (n * np.sqrt(sums[1] / n)); gp = k * d; ga = np.abs(gp)
    elif loss_type == L.LOSS_L1_SMOOTH:
        gp = np.clip(d, -1, 1) / n; ga = np.abs(gp)
    elif loss_type == L.LOSS_NCC:
        pp, tt = sums[4], sums[5]
        cc = sums[3] / np.sqrt(pp * tt)
        ncc = np.sqrt(max(1e-30, 2 - 2 * cc))
        a, b = -1.0 / (ncc * np.sqrt(pp * tt)), cc / (ncc * pp)
        gp = a * tg + b * pv; ga = np.abs(a * tg) + np.abs(b * pv)
    else:
        gp = dpred_cpu.astype(np.float64); ga = np.abs(gp)
    got, mag = np.zeros((len(c.sel), 9)), np.zeros((len(c.sel), 9))
    for s0 in range(0, len(c.sel), 16):
        sl = slice(s0, s0 + 16)
        tt_ = {k: (v[sl] if isinstance(v, np.ndarray) and v.shape[:1] == (len(c.sel),) else v) for k, v in t.items()}
        terms, m = R.bwd_terms(c.I_cpu[sl], tt_, gp[sl], ga[sl])
        got[sl] = terms.sum(axis=(1, 2)); mag[sl] = m.sum(axis=(1, 2))
    return got, mag


def _bwd_tau(c):
    """Relative rounding bound of dH' against sum |term|: ~16 fp32 roundings per term, 4 pixels per thread, a 256-thread
    shuffle tree (10 levels), then one float atomic per CTA of the sample."""
    ctas = ((c.pw + 127) // 128) * ((c.ph + 7) // 8)
    return (16 + 4 + 10 + ctas) * U


LOSSES = ["L1", "REC", "L1_SMOOTH", "NCC", "CUSTOM"]


def test_warp_backward_all_losses_on_restated_gates(udh, case):
    L = udh.lib
    c = case
    sums = c.sums.cpu().numpy()
    tau = _bwd_tau(c)
    sel_t = torch.tensor(c.sel, device="cuda")
    print("\n[%s] backward, tau = %.2e" % (c.name, tau))
    for name in LOSSES:
        lt = getattr(L, "LOSS_" + name)
        dpred = udh.ops.ssim_backward(c.pred, c.I2, c.pw, c.ph) if name == "CUSTOM" else None
        dH = torch.empty(c.B, 9, device="cuda"); scratch = torch.empty(c.B * 9, device="cuda")
        stride = 0 if c.idx is None else (c.idx.stride(0) if c.idx.dim() > 1 else 1)
        L.check(L.lib.udh_warp_loss_bwd_ex(_p(c.I), c.C, IMG_H, IMG_W, _p(c.H), _p(c.I2), _p(c.idx), stride, c.pw, c.ph, lt,
                                          _p(c.sums), _p(dpred), ctypes.c_float(1.0), _p(dH), _p(scratch), c.B,
                                          udh.ops._stream()), "bwd")
        torch.cuda.synchronize()
        dHn = scratch.reshape(c.B, 9)[sel_t].cpu().numpy().astype(np.float64)
        dpc = dpred[sel_t].cpu().numpy() if dpred is not None else None
        ref, mag = _bwd_reference(c, lt, L, sums, dpc)
        ratio = np.abs(dHn - ref) / np.maximum(mag, 1e-300)
        _report("%s dH' |err| / sum|term|" % name, ratio.max(), tau)
        assert (np.abs(dHn - ref) <= tau * mag).all(), (name, np.unravel_index(ratio.argmax(), ratio.shape), ratio.max())
        # the conjugation of the kernel's own dH'
        conj, cmag = R.conj_bwd(scratch.reshape(c.B, 9).cpu().numpy(), IMG_W, IMG_H)
        err = np.abs(dH.cpu().numpy() - conj)
        _report("%s dH = conj(dH') |err| / magnitude" % name, (err / np.maximum(cmag, 1e-300)).max(), 4 * U)
        assert (err <= 4 * U * cmag).all()
        if name in ("L1", "REC", "L1_SMOOTH") and c.B <= 129:
            Hg = c.H.reshape(c.B, 3, 3).clone().requires_grad_(True)
            udh.ops.warp_photo_loss(Hg, c.I, c.I2, c.idx, c.pw, c.ph, lt).backward()
            cref, _ = R.conj_bwd(ref, IMG_W, IMG_H)
            _, cb = R.conj_bwd(tau * mag, IMG_W, IMG_H)
            _, cm = R.conj_bwd(mag, IMG_W, IMG_H)
            e = np.abs(Hg.grad.cpu().numpy().reshape(c.B, 9)[c.sel] - cref)
            _report("%s autograd dH vs conj(fp64 dH')" % name, (e / np.maximum(cb + 4 * U * cm, 1e-300)).max(), 1.0)
            assert (e <= cb + 4 * U * cm).all()


# ------------------------------------------------------------------------------------------------ b. forward pixels
def test_warp_forward_pixels_within_rcp_box(udh, case):
    c = case
    t = c.t
    pred = c.pred_cpu[c.sel]
    dx, dy = R.forward_coord_delta(t, IMG_W, IMG_H)
    xc, yc = R.box_candidates(t["x"], dx), R.box_candidates(t["y"], dy)
    bidx = np.arange(len(c.sel))[:, None, None]
    lo = np.full(pred.shape, np.inf); hi = np.full(pred.shape, -np.inf)
    slack = np.zeros(pred.shape); allzero = np.ones(pred.shape, bool); yclip = np.ones(pred.shape, bool)
    for i in range(4):
        for j in range(4):
            tap = R.tap_from_xy(xc[..., i], yc[..., j], IMG_W, IMG_H)
            v = R.sample_gray(c.I_cpu, tap, bidx).astype(np.float64)
            lo = np.fmin(lo, v); hi = np.fmax(hi, v)
            slack = np.fmax(slack, R.blend_magnitude(c.I_cpu, tap, bidx))
            allzero &= v == 0
            yclip &= tap["y0"] == tap["y1"]
    slack = (8 + 2 * c.C) * U * slack
    p = pred.astype(np.float64)
    below, above = np.maximum(lo - slack - p, 0), np.maximum(p - hi - slack, 0)
    fin = np.isfinite(t["pv"])
    width = np.where(fin, hi - lo + slack, 0)
    ident = (pred == t["pv"]).mean()
    sign_f = np.sign(pred - c.I2_cpu[c.sel]); sign_b = np.sign(t["pv"] - c.I2_cpu[c.sel])
    print("\n[%s] forward: %.4f of pixels bit-identical to the restated IEEE value, %d pixels where sign(pred - I2) differs "
          "from the backward's, %d pixels black over the whole box" % (c.name, ident, int((sign_f != sign_b).sum()), int(allzero.sum())))
    _report("pred outside the rcp box range (px value)", max(below[fin].max(), above[fin].max()), 0.0)
    _report("widest box range + slack", width.max(), np.inf)
    assert (below[fin] == 0).all() and (above[fin] == 0).all()
    # the black border.  Where y clips over the whole box the taps pair up (Ia == Ib, wb == -wa; Ic == Id, wd == -wc) and
    # the blend is exactly 0.  Where only x clips, fl(wa*Ia + wb*Ib) - wa*Ia need not be wb*Ib: a residue of the blend's
    # rounding can remain at the forward's coordinates even where the restatement is 0 over the whole box (warp.cu
    # bilinear_rn)
    yz = yclip & fin
    assert (pred[yz] == 0).all(), int((pred[yz] != 0).sum())
    res = np.abs(p[allzero])
    print("  y-clipped pixels: %d, all exactly 0; black-border pixels with a nonzero residue: %d, largest %.3e (bound %.3e)"
          % (int(yz.sum()), int((res > 0).sum()), res.max() if res.size else 0.0, slack[allzero].max() if res.size else 0.0))
    assert (res <= slack[allzero]).all()


# ------------------------------------------------------------------------------------------------ c. sums and finalize
def _sum_refs(p, t):
    p = p.astype(np.float64); t = t.astype(np.float64)
    d32 = (p.astype(f32) - t.astype(f32)).astype(np.float64)
    ad = np.abs(d32)
    hub = np.where(ad < 1, 0.5 * d32 * d32, ad - 0.5)
    terms = [ad, d32 * d32, hub, p * t, p * p, t * t]
    return np.array([x.sum() for x in terms]), np.array([np.abs(x).sum() for x in terms])


def test_warp_forward_sums_and_finalize(udh, case):
    L = udh.lib
    c = case
    sums = c.sums.cpu().numpy()
    ref, mag = _sum_refs(c.pred_cpu, c.I2_cpu)
    quads = c.ph * c.pw // 4
    k = -(-quads // 256)                                       # quads per thread with the smallest grid (X = 1)
    tau = (4 * k + 8) * U
    r = np.abs(sums[:6] - ref) / mag
    print("\n[%s] sums" % c.name)
    _report("six sums |err| / sum|term| (worst of six)", r.max(), tau)
    assert (r <= tau).all(), r
    # the l1-only template (bench.py's configs[3] kernel) against the full one and against fp64
    s1 = torch.zeros(L.NSUMS, device="cuda", dtype=torch.float64)
    stride = 0 if c.idx is None else (c.idx.stride(0) if c.idx.dim() > 1 else 1)
    L.check(L.lib.udh_warp_loss_fwd_ex(_p(c.I), c.C, IMG_H, IMG_W, _p(c.H), _p(c.I2), _p(c.idx), stride, c.pw, c.ph, None,
                                       _p(s1), 0, c.B, udh.ops._stream()), "fwd_ex")
    a1 = s1[0].item()
    _report("l1-only template sum |d| vs fp64 / sum|term|", abs(a1 - ref[0]) / mag[0], tau)
    assert abs(a1 - ref[0]) <= tau * mag[0]
    if c.name == "full_B64_C1":
        # bench.py's configs[3] shape: both templates run the same grid there, so their fp32 per-thread partials are the
        # same and only the order of the fp64 atomics differs.  (Where the two templates' occupancies differ, e.g. C = 3
        # at B = 128, they pick different grids X and agree only to the fp32 partials' bound above.)
        _report("l1-only template sum |d| vs full template (relative)", abs(a1 - sums[0]) / sums[0], 1e-12)
        assert abs(a1 - sums[0]) <= 1e-12 * sums[0]
    assert (s1[1:].cpu().numpy() == 0).all()
    # finalisation from the same sums (SSIM slot filled by the kernel's own ssim_fwd)
    n, n_ssim = float(c.B * c.pw * c.ph), float(c.B * (c.pw - 2) * (c.ph - 2))
    out = udh.ops.photo_losses(c.pred, c.I2, c.sums, c.pw, c.ph, c.B).cpu().numpy()
    s = c.sums.cpu().numpy()
    cc = s[3] / np.sqrt(s[4] * s[5])
    want = {L.L_REC: np.sqrt(s[1] / n), L.L_SSIM: s[6] / n_ssim, L.L_L1: s[0] / n, L.L_L1_SMOOTH: s[2] / n,
            L.L_NCC: np.sqrt(max(0.0, 2 - 2 * cc))}
    worst = 0.0
    for slot, w in want.items():
        e = abs(float(out[slot]) - w) / max(abs(w), 1e-30)
        worst = max(worst, e)
        tol = 2 * U + (4 * 2.0 ** -53 / max(2 - 2 * cc, 1e-30) if slot == L.L_NCC else 0)
        assert e <= tol, (slot, out[slot], w)
    _report("finalize relative error (worst slot)", worst, 2 * U)


# ------------------------------------------------------------------------------------------------ d. SSIM
C1, C2 = float(f32(0.01) * f32(0.01)), float(f32(0.03) * f32(0.03))   # the kernel's fp32 constants


def _ssim_stats(x, y):
    """3x3 VALID window sums of x, y, x^2, y^2, xy and of |xy| in fp64: [S, oh, ow] each."""
    def box(a):
        s = 0
        for dy in range(3):
            for dx in range(3):
                s = s + a[:, dy:dy + a.shape[1] - 2, dx:dx + a.shape[2] - 2]
        return s
    return box(x), box(y), box(x * x), box(y * y), box(x * y), box(np.abs(x)), box(np.abs(y)), box(np.abs(x * y))


def _L_of(mx, my, vx, vy, vxy):
    n = (2 * mx * my + C1) * (2 * vxy + C2)
    d = (mx * mx + my * my + C1) * (vx + vy + C2)
    return (1 - n / d) / 2


def _dS_of(mx, my, vx, vy, vxy, xi, yi):
    k = 1.0 / 9
    A1, A2, B1, B2 = 2 * mx * my + C1, 2 * vxy + C2, mx * mx + my * my + C1, vx + vy + C2
    S = A1 * A2 / (B1 * B2)
    dA1, dA2, dB1, dB2 = 2 * my * k, 2 * (yi - my) * k, 2 * mx * k, 2 * (xi - mx) * k
    dS = (dA1 * A2 + A1 * dA2) / (B1 * B2) - S * (dB1 * B2 + B1 * dB2) / (B1 * B2)
    mag = (abs(dA1 * A2) + abs(A1 * dA2)) / abs(B1 * B2) + abs(S) * (abs(dB1 * B2) + abs(B1 * dB2)) / abs(B1 * B2)
    return dS, mag


def _ssim_errors(sx, sy, sxx, syy, sxy, ax, ay, axy):
    """fp64 window statistics and first-order bounds of the kernel's fp32 error in each (9-term fp32 sums, * fp32(1/9),
    sigma^2 = E[x^2] - mu^2 with its cancellation)."""
    k = 1.0 / 9
    mx, my = sx * k, sy * k
    st = [mx, my, sxx * k - mx * mx, syy * k - my * my, sxy * k - mx * my]
    emx, emy = 12 * U * ax * k, 12 * U * ay * k
    err = [emx, emy,
           12 * U * sxx * k + 2 * abs(mx) * emx + 3 * U * mx * mx,
           12 * U * syy * k + 2 * abs(my) * emy + 3 * U * my * my,
           12 * U * axy * k + abs(mx) * emy + abs(my) * emx + 3 * U * abs(mx * my)]
    return st, err


def _ssim_inputs(udh, kind):
    """(pred, I2) [B,128,128] on the device.  'warp_*': the kernel's own pred of a warp case (black border, a horizon,
    translations); 'noise': pred ~ N(0,1) and I2 = 0.6 pred + 0.8 N(0,1), well-conditioned windows whose L lies far from
    the clip points, so that the bound of the forward's sum is tight."""
    if kind == "noise":
        g = torch.Generator(device="cuda"); g.manual_seed(11)
        x = torch.randn(129, 128, 128, device="cuda", generator=g)
        y = 0.6 * x + 0.8 * torch.randn(129, 128, 128, device="cuda", generator=g)
        return x.contiguous(), y.contiguous()
    B, C, origins, idx_kind = {"warp_B1": (1, 1, "rand", "table"), "warp_B128_C1": (128, 1, "rand", "table"),
                               "warp_B129_C3_extreme": (129, 3, "extreme", "origin")}[kind]
    c = _inputs(udh, B, C, 128, 128, origins, idx_kind, seed=B * 7 + C)
    pred, _ = udh.ops.warp_loss_forward(c.I, c.H, c.I2, c.idx, 128, 128)
    return pred[..., 0].contiguous(), c.I2


def _window_L_bound(st, err):
    """fp64 L per window and a bound of the kernel's |L_fp32 - L| (first order in the statistics' errors, doubled, plus
    the rounding of the final expression)."""
    Lw = _L_of(*st)
    eL = sum(np.abs(_L_of(*[s + (e if i == j else 0) for j, s in enumerate(st)])
                    - _L_of(*[s - (e if i == j else 0) for j, s in enumerate(st)])) / 2 for i, e in enumerate(err))
    return Lw, 2 * eL + 10 * U * (1 + np.abs(Lw))


@pytest.mark.parametrize("kind", ["warp_B1", "warp_B128_C1", "warp_B129_C3_extreme", "noise"])
def test_ssim_forward_and_backward_vs_fp64(udh, kind):
    pred, I2 = _ssim_inputs(udh, kind)
    B, ph, pw = pred.shape
    x = pred.cpu().numpy().astype(np.float64); y = I2.cpu().numpy().astype(np.float64)
    sums = torch.zeros(8, device="cuda", dtype=torch.float64)
    udh.lib.check(udh.lib.lib.udh_ssim_fwd(_p(pred), _p(I2), pw, ph, _p(sums), B, udh.ops._stream()), "ssim_fwd")
    dX = udh.ops.ssim_backward(pred, I2, pw, ph).cpu().numpy().astype(np.float64)
    inv_n = float(f32(1) / (f32(B) * f32(pw - 2) * f32(ph - 2)))
    # forward: the kernel sums clip(L_fp32) in fp64, so its error is the sum of the per-window errors.  clip is 1-Lipschitz,
    # and a window whose whole error interval lies beyond a clip point contributes nothing.
    ref = bound = 0.0
    for s0 in range(0, B, 32):
        st, err = _ssim_errors(*_ssim_stats(x[s0:s0 + 32], y[s0:s0 + 32]))
        Lw, eL = _window_L_bound(st, err)
        ref += np.clip(Lw, 0, 1).sum()
        bound += (np.clip(Lw + eL, 0, 1) - np.clip(Lw - eL, 0, 1)).sum()
    e = abs(sums[6].item() - ref)
    print("\n[ssim %s] sum of L = %.6e" % (kind, ref))
    _report("ssim_fwd sum |err| / sum", e / ref, bound / ref)
    assert e <= bound
    if kind == "noise":
        assert bound <= 3e-5 * ref                              # well-conditioned windows: the bound itself is tight
    # backward per pixel on the restated samples
    sel = _sel(B)
    xs, ys = x[sel], y[sel]
    st, err = _ssim_errors(*_ssim_stats(xs, ys))
    Lw, eL = _window_L_bound(st, err)
    amb = (np.abs(Lw) <= eL) | (np.abs(Lw - 1) <= eL)          # either clip decision is right within rounding
    on = (Lw > 0) & (Lw < 1)
    g = np.zeros_like(xs); gb = np.zeros_like(xs)
    oh, ow = Lw.shape[1], Lw.shape[2]
    for dy in range(3):
        for dx in range(3):
            xi, yi = xs[:, dy:dy + oh, dx:dx + ow], ys[:, dy:dy + oh, dx:dx + ow]
            dS, mag = _dS_of(*st, xi, yi)
            edS = sum(np.abs(_dS_of(*[s + (e if i == j else 0) for j, s in enumerate(st)], xi, yi)[0]
                             - _dS_of(*[s - (e if i == j else 0) for j, s in enumerate(st)], xi, yi)[0]) / 2
                      for i, e in enumerate(err))
            g[:, dy:dy + oh, dx:dx + ow] += np.where(on, -0.5 * dS, 0)
            gb[:, dy:dy + oh, dx:dx + ow] += (0.5 * (2 * edS + 20 * U * mag) + np.where(amb, 0.5 * np.abs(dS), 0)
                                               + 9 * U * 0.5 * np.abs(dS))
    got = dX[sel]
    bb = inv_n * gb + U * np.abs(g * inv_n) + 1e-30
    r = np.abs(got - g * inv_n) / bb
    _report("ssim_bwd per pixel |err| / bound", r.max(), 1.0)
    assert (r <= 1).all(), (np.unravel_index(r.argmax(), r.shape), r.max())


# ------------------------------------------------------------------------------------------------ e. bit-exact resamplers
def test_transformer_bit_identical(udh):
    rng = np.random.default_rng(4)
    for (B, H, W, C, oh, ow) in ((3, 24, 32, 3, 24, 32), (2, 240, 320, 1, 128, 160), (4, 60, 80, 3, 97, 131)):
        Uimg = rng.normal(size=(B, H, W, C)).astype(f32)
        th = np.tile(np.eye(3, dtype=f32).reshape(1, 9), (B, 1))
        th[1:] = (th[1:] + rng.normal(0, 0.05, size=(B - 1, 9))).astype(f32)
        th[-1, 6:8] = [0.9, -0.4]                               # horizon inside the output grid
        out, _ = udh.ops.transformer(torch.tensor(Uimg).cuda(), torch.tensor(th).cuda(), (oh, ow))
        ref = R.transformer(Uimg, th, oh, ow)
        got = out.cpu().numpy()
        same = (got == ref) | (np.isnan(got) & np.isnan(ref))
        assert same.all(), (B, H, W, C, int((~same).sum()))
    print("\n  transformer: bit-identical on every element")


def test_warp_image_u8_bit_identical(udh):
    L = udh.lib
    B = 24
    I_u8 = torch.empty(B, IMG_H, IMG_W, 3, device="cuda", dtype=torch.uint8)
    pts1 = torch.empty(B, 8, device="cuda"); gt = torch.empty(B, 8, device="cuda")
    L.check(L.lib.udh_synth_scene_u8(_p(I_u8), _p(pts1), _p(gt), B, IMG_H, IMG_W, 128, 45, 1234, udh.ops._stream()), "scene")
    H = udh.ops.dlt_forward(pts1, gt).reshape(B, 9).clone()
    rng = np.random.default_rng(5)
    hand = [[1, 0, 0, 0, 1, 0, 0, 0, 1], [1, 0, 7, 0, 1, -13, 0, 0, 1], [0.5, 0, 0, 0, 0.5, 0, 0, 0, 1],
            [1, 0.1, 0, -0.1, 1, 0, -1 / 160.3, 1e-4, 1], [2.5, 0.3, -100, 0.1, 2.2, -80, 1e-3, -2e-3, 1],
            [1, 0, 400, 0, 1, 0, 0, 0, 1]]
    H[:len(hand)] = torch.tensor(np.array(hand, f32)).cuda()
    H[len(hand):len(hand) + 4] = (H[len(hand):len(hand) + 4] * (1 + 1e-2 * torch.tensor(rng.normal(size=(4, 9)).astype(f32)).cuda()))
    H = H.contiguous()
    out = torch.empty_like(I_u8)
    L.check(L.lib.udh_warp_image_u8(_p(I_u8), _p(H), _p(out), B, IMG_H, IMG_W, udh.ops._stream()), "warp_u8")
    ref = R.warp_image_u8(I_u8.cpu().numpy(), H.cpu().numpy())
    got = out.cpu().numpy()
    assert (got == ref).all(), int((got != ref).sum())
    print("\n  warp_image_u8: bit-identical on %d pixels" % got.size)


# ------------------------------------------------------------------------------------------------ f. DLT
DLT_C = 64.0


def _dlt_inputs(B, kind, rng):
    x0 = rng.integers(45, 148, size=B); y0 = rng.integers(45, 68, size=B)
    pts1 = np.stack([x0, y0, x0 + 128, y0, x0 + 128, y0 + 128, x0, y0 + 128], 1).astype(f32)
    if kind == "zero":
        h4p = np.zeros((B, 8), f32)
    elif kind == "int":
        h4p = rng.integers(-45, 46, size=(B, 8)).astype(f32)
    elif kind == "real":
        h4p = rng.uniform(-45, 45, size=(B, 8)).astype(f32)
    else:                                                        # near-degenerate: corner 2 pulled onto the line 1-3
        h4p = rng.uniform(-10, 10, size=(B, 8)).astype(f32)
        p = pts1 + h4p
        eps = 10.0 ** rng.uniform(-4, 0, size=B)
        tgt = 0.5 * (p[:, 0:2] + p[:, 4:6]) + eps[:, None] * rng.normal(size=(B, 2))
        h4p[:, 2:4] = (tgt - pts1[:, 2:4]).astype(f32)
    return pts1, h4p


@pytest.mark.parametrize("B", [1, 3, 5, 128, 129, 1000, 4096])
def test_dlt_forward_backward_vs_fp64(udh, B):
    rng = np.random.default_rng(B)
    print()
    for kind in ("zero", "int", "real", "degenerate"):
        pts1, h4p = _dlt_inputs(B, kind, rng)
        Hc = udh.ops.dlt_forward(torch.tensor(pts1).cuda(), torch.tensor(h4p).cuda())
        H = Hc.reshape(B, 9).cpu().numpy()
        ref, cond = R.dlt_fwd(pts1, h4p)
        assert (H[:, 8] == 1).all()
        scale = np.abs(ref).max(1, keepdims=True)
        half_ulp = np.spacing(np.abs(ref).astype(f32)).astype(np.float64) / 2
        bound = half_ulp + DLT_C * cond[:, None] * R.U64 * scale
        r = np.abs(H - ref) / bound
        _report("DLT fwd B=%d %s |err| / bound (max cond %.1e)" % (B, kind, cond.max()), r.max(), 1.0)
        assert (r <= 1).all(), (kind, np.unravel_index(r.argmax(), r.shape))
        dH = rng.normal(size=(B, 9)).astype(f32)
        dh = udh.ops.dlt_backward(torch.tensor(pts1).cuda(), torch.tensor(h4p).cuda(), Hc, torch.tensor(dH).reshape(B, 3, 3).cuda()).cpu().numpy()
        bref, bscale, cond_b = R.dlt_bwd(pts1, h4p, H, dH)
        bb = np.spacing(np.abs(bref).astype(f32)).astype(np.float64) / 2 + DLT_C * cond_b[:, None] * R.U64 * bscale[:, None]
        rb = np.abs(dh - bref) / bb
        _report("DLT bwd B=%d %s |err| / bound" % (B, kind), rb.max(), 1.0)
        assert (rb <= 1).all(), (kind, np.unravel_index(rb.argmax(), rb.shape))
    print("  DLT constant c = %g (bound = half an fp32 ulp + c * cond(A) * 2^-53 * max|.|)" % DLT_C)


# ------------------------------------------------------------------------------------------------ g. udh_h4p_loss
def _h4p_ref(pred, gt):
    d = pred.astype(np.float64) - gt.astype(np.float64)
    bh = np.sqrt((d * d).mean(1)); ih = np.sqrt((gt.astype(np.float64) ** 2).mean(1))
    return d, bh, ih


@pytest.mark.parametrize("B", [1, 255, 256, 257, 4096])
def test_h4p_loss_vs_fp64(udh, B):
    L = udh.lib
    rng = np.random.default_rng(B + 7)
    gt = rng.integers(-45, 46, size=(B, 8)).astype(f32)
    gt[::11] = 0                                               # identity error 0: a failure whatever pred is
    pred = (gt + rng.normal(0, 20, size=(B, 8))).astype(f32)
    cases = {"noise": pred, "zero": np.zeros_like(gt), "exact": gt.copy()}
    print()
    for name, pr in cases.items():
        m, per, dp = udh.ops.h4p_loss(torch.tensor(pr).cuda(), torch.tensor(gt).cuda(), want_grad=True, want_per_sample=True)
        m, per, dp = m.cpu().numpy(), per.cpu().numpy(), dp.cpu().numpy()
        d, bh, ih = _h4p_ref(pr, gt)
        r = np.abs(per - bh) / np.maximum(bh * 8 * U, 1e-30)
        assert (np.abs(per - bh) <= 8 * U * bh).all(), (name, r.max())
        fail = bh >= ih
        tie = np.abs(bh - ih) <= 16 * U * np.maximum(bh, ih)
        hl = np.sqrt((d * d).mean())
        bounded = np.where(fail, ih, bh).mean()
        ace = np.sqrt((d.reshape(B, 4, 2) ** 2).sum(2)).mean()
        assert abs(m[L.M_H_LOSS] - hl) <= 8 * U * hl
        assert abs(m[L.M_BOUNDED_H_LOSS] - bounded) <= 8 * U * bounded + 16 * U * ih[tie].sum() / B
        assert abs(m[L.M_ACE] - ace) <= 8 * U * ace
        assert fail[~tie].sum() <= m[L.M_NUM_FAIL] <= fail[~tie].sum() + tie.sum()
        k = 1.0 / (8 * B * float(m[L.M_H_LOSS])) if m[L.M_H_LOSS] > 0 else 0.0
        assert (np.abs(dp - d * k) <= 8 * U * np.abs(d * k)).all()
        if name == "zero":                                     # pred = 0: batch == identity error exactly -> every sample fails
            assert m[L.M_NUM_FAIL] == B and abs(m[L.M_BOUNDED_H_LOSS] - ih.mean()) <= 8 * U * ih.mean()
        if name == "exact":
            assert m[L.M_H_LOSS] == 0 and (dp == 0).all() and not np.isnan(dp).any()
            assert m[L.M_NUM_FAIL] == (gt == 0).all(1).sum()  # bh = 0 >= ih only where gt = 0
        else:
            zero_rows = (gt == 0).all(1)
            assert (fail[zero_rows]).all()
        _report("h4p B=%d %s per-sample |err| / (8 u |bh|), ties %d" % (B, name, int(tie.sum())), r.max(), 1.0)


# ------------------------------------------------------------------------------------------------ h. the chain inside the step
def _check_chain(label, batch, ox, oy, r, B, P, C):
    """The dH and dh4p a path hands to the CNN backward against references built from that path's own H_mat, pred_h4p and
    the inputs: the DLT forward within f's bound, dH' (when the path exposes it) within a's, dH against the fp64
    conjugation, dh4p = dlt_bwd of the path's own dH within f's bound."""
    pts1 = batch["pts1"].cpu().numpy()
    h4p, H, dH, dh4p = (r[k].cpu().numpy().reshape(B, -1) for k in ("h4p", "H", "dH", "dh4p"))
    Href, cond = R.dlt_fwd(pts1, h4p)
    assert (H[:, 8] == 1).all()
    hb = np.spacing(np.abs(Href).astype(f32)).astype(np.float64) / 2 + DLT_C * cond[:, None] * R.U64 * np.abs(Href).max(1, keepdims=True)
    _report("%s: H_mat vs fp64 DLT of its own pred_h4p / bound" % label, (np.abs(H - Href) / hb).max(), 1.0)
    assert (np.abs(H - Href) <= hb).all()
    # dH' on the restated gates of the path's own H (l1_loss: sign(d) / (B P P), upstream 1)
    sel = _sel(B)
    I_cpu = batch["I_aug"][torch.tensor(sel, device="cuda")].cpu().numpy()
    t = R.warp_window(I_cpu, H[sel], ox[sel], oy[sel], P, P)
    tg = batch["I2_aug"].reshape(B, P, P).cpu().numpy()[sel]
    d = (t["pv"] - tg).astype(f32).astype(np.float64)
    n = float(B * P * P)
    terms, mag = R.bwd_terms(I_cpu, t, np.sign(d) / n, np.full(d.shape, 1.0 / n))
    ref, mag = terms.sum(axis=(1, 2)), mag.sum(axis=(1, 2))
    tau = (16 + 4 + 10 + 16) * U                                # as _bwd_tau for the 128 window: 16 CTAs per sample
    if "dHn" in r:
        dHn = r["dHn"].cpu().numpy().reshape(B, 9)
        ratio = np.abs(dHn[sel] - ref) / mag
        _report("%s: dH' |err| / sum|term|" % label, ratio.max(), tau)
        assert (ratio <= tau).all()
        conj, cmag = R.conj_bwd(dHn, IMG_W, IMG_H)
        _report("%s: dH = conj(own dH') |err| / magnitude" % label, (np.abs(dH - conj) / cmag).max(), 4 * U)
        assert (np.abs(dH - conj) <= 4 * U * cmag).all()
    cref, _ = R.conj_bwd(ref, IMG_W, IMG_H)
    _, cb = R.conj_bwd(tau * mag, IMG_W, IMG_H)
    _, cm = R.conj_bwd(mag, IMG_W, IMG_H)
    e = np.abs(dH[sel] - cref)
    _report("%s: dH vs conj(fp64 dH') / bound" % label, (e / (cb + 4 * U * cm)).max(), 1.0)
    assert (e <= cb + 4 * U * cm).all()
    bref, bscale, cond_b = R.dlt_bwd(pts1, h4p, H, dH)
    bb = np.spacing(np.abs(bref).astype(f32)).astype(np.float64) / 2 + DLT_C * cond_b[:, None] * R.U64 * bscale[:, None]
    _report("%s: dh4p vs fp64 dlt_bwd of its own H, dH / bound" % label, (np.abs(dh4p - bref) / bb).max(), 1.0)
    assert (np.abs(dh4p - bref) <= bb).all()


@pytest.mark.parametrize("variant", ["gray_origin", "rgb_table"])
def test_l1_step_chain_vs_restated_references(udh, variant):
    """The default l1_loss step at B = 128 in the two-limb mode, once as the one-call udh_step_forward_backward and once as
    engine.forward + engine.backward through the individual entry points."""
    from unsuperviseddeephomographyral2018_b200 import engine, params
    L = udh.lib
    B, P, rgb = 128, 128, variant == "rgb_table"
    fb = udh.synthetic.make_batch_fast(B, seed=23, want_rgb=rgb)
    origin = fb["patch_indices"].cpu().numpy().astype(np.int64)
    ox, oy = origin % IMG_W, origin // IMG_W
    batch = {k: fb[k].contiguous() for k in ("I1_aug", "I2_aug", "pts1", "gt")}
    batch["I_aug"] = (fb["I_aug_rgb"] if rgb else fb["I_aug"]).contiguous()
    if rgb:                                                     # the full [B, P*P] index table (stride P*P)
        yy, xx = np.meshgrid(np.arange(P), np.arange(P), indexing="ij")
        batch["patch_indices"] = torch.tensor(((yy[None] + oy[:, None, None]) * IMG_W + xx[None] + ox[:, None, None])
                                              .reshape(B, -1).astype(np.int32)).cuda()
    else:                                                       # the fast generator's origins, stride 1
        batch["patch_indices"] = fb["patch_indices"]
    eng = engine.HomographyEngine(B, numeric="bf16x3", seed=None, loss_type="l1_loss")
    eng.load_flat(params.init_flat_large(3))                    # |pred_h4p| of tens of pixels
    # one-call step, forward + backward only (no optimiser update, so the second path sees the same weights and seed)
    a = eng._fill_args(batch, True)
    L.check(L.lib.udh_step_forward_backward(ctypes.byref(a), L.STEP_ALL, udh.ops._stream()), "udh_step_forward_backward")
    sb = eng._sb
    step = {"h4p": sb["h4p"].clone(), "H": sb["H"].clone(), "dHn": sb["scratch"].clone(), "dH": sb["dH"].clone(),
            "dh4p": sb["dh4p"].clone()}
    eng.grads.zero_()
    out = eng.forward(batch, train=True)
    eng.backward(batch, out)
    sep = {"h4p": out["pred_h4p"], "H": out["H_mat"], "dH": out["_dH"], "dh4p": out["_dh4p"]}
    torch.cuda.synchronize()
    assert float(step["h4p"].abs().max()) > 10.0
    print("\n[step chain %s]" % variant)
    _check_chain("one-call step", batch, ox, oy, step, B, P, 3 if rgb else 1)
    _check_chain("engine.backward", batch, ox, oy, sep, B, P, 3 if rgb else 1)
