"""CPU checks of oracle/warp_fp32.py, the NumPy restatement of the photometric kernels' fp32 arithmetic that
tests/test_gpu_photometric.py compares the kernels with."""
from fractions import Fraction

import numpy as np
import torch

from oracle import oracle as O
from oracle import warp_fp32 as R

f32 = np.float32


def _round_fraction_to_f32(q):
    """Round a Fraction to the nearest fp32 (ties to even), exactly."""
    if q == 0:
        return f32(0)
    s = -1 if q < 0 else 1
    q = abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if Fraction(2) ** e > q:
        e -= 1
    e = max(e, -126)                                    # subnormal range keeps the exponent of 2^-126
    scale = Fraction(2) ** (e - 23)
    m = q / scale
    n = m.numerator // m.denominator
    rem = m - n
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and n % 2 == 1):
        n += 1
    return f32(s * float(n * scale))


def _exact_fma(a, b, c):
    return _round_fraction_to_f32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def test_fmaf32_random_triples_exact():
    rng = np.random.default_rng(0)
    n = 100_000
    a = (rng.standard_normal(n) * np.exp2(rng.integers(-20, 20, n))).astype(f32)
    b = (rng.standard_normal(n) * np.exp2(rng.integers(-20, 20, n))).astype(f32)
    c = (-(a.astype(np.float64) * b) * (1 + rng.standard_normal(n) * np.exp2(rng.integers(-30, 0, n)))).astype(f32)
    c[::3] = (rng.standard_normal(n)[::3] * 10).astype(f32)
    got = R.fmaf32(a, b, c)
    bad = [i for i in range(n) if got[i] != _exact_fma(a[i], b[i], c[i])]
    assert not bad, bad[:5]


def test_fmaf32_midpoints_need_twosum():
    # a*b = 1 + 2^-24 + 2^-70-ish residue: the fp64 sum lands exactly on the fp32 midpoint 1 + 2^-24, and only the
    # residue below fp64's precision says that the exact result lies above it
    a = f32(1 + 2.0 ** -12)
    b = f32(1 + 2.0 ** -12)                             # a*b = 1 + 2^-11 + 2^-24 exactly
    c = f32(-(2.0 ** -11))                              # a*b + c = 1 + 2^-24: an exact midpoint, ties to even -> 1
    assert R.fmaf32(a, b, c) == _exact_fma(a, b, c) == f32(1)
    # a*b = 1 + 2^-11 + 2^-24 is an fp32 midpoint; c = 2^-80 is lost in the fp64 sum, so rounding that sum to fp32
    # ties to even (1 + 2^-11) while the exact a*b + c lies above the midpoint (1 + 2^-11 + 2^-23)
    c2 = f32(2.0 ** -80)
    exact = _exact_fma(a, b, c2)
    naive = f32(float(a) * float(b) + float(c2))
    assert exact == f32(1 + 2.0 ** -11 + 2.0 ** -23) and naive == f32(1 + 2.0 ** -11), (exact, naive)
    assert R.fmaf32(a, b, c2) == exact
    for cc in (f32(0), -c2):
        assert R.fmaf32(a, b, cc) == _exact_fma(a, b, cc) == f32(1 + 2.0 ** -11)
    # constructed midpoints s (1 + 2^-e1)(1 + 2^-(24-e1)) 2^j in many binades, with residues of both signs and none
    for e1 in range(1, 24):
        for j in (-40, -3, 0, 5, 30):
            for s in (1.0, -1.0):
                aa = f32(s * (1 + 2.0 ** -e1) * 2.0 ** j); bb = f32(1 + 2.0 ** -(24 - e1))
                for k in (0, 60, 75, 100):
                    for sg in (1.0, -1.0):
                        cc = f32(sg * 2.0 ** (j - k)) if k else f32(0)
                        assert R.fmaf32(aa, bb, cc) == _exact_fma(aa, bb, cc), (aa, bb, cc)


def _coords64(H, W, Hh, ox, oy, pw, ph):
    """fp64 source coordinates of the windows (homography_model.py:252-269 in exact-ish arithmetic)."""
    M, Mi = O.norm_matrices(W, Hh, torch.float64)
    Hn = (Mi.numpy() @ np.asarray(H, np.float64).reshape(-1, 3, 3) @ M.numpy())
    xt = -1.0 + (np.asarray(ox)[:, None, None] + np.arange(pw)[None, None, :]) * (2.0 / (W - 1))
    yt = -1.0 + (np.asarray(oy)[:, None, None] + np.arange(ph)[None, :, None]) * (2.0 / (Hh - 1))
    T = [Hn[:, r, 0, None, None] * xt + Hn[:, r, 1, None, None] * yt + Hn[:, r, 2, None, None] for r in range(3)]
    ts = np.where(np.abs(T[2]) >= 1e-7, T[2], T[2] + 1e-6)
    return (T[0] / ts + 1) * W / 2, (T[1] / ts + 1) * Hh / 2


def test_restated_sampler_matches_fp64_transform():
    B = 3
    batch = O.make_batch(5, B)
    h4p = batch["gt"] + torch.tensor(np.random.default_rng(5).normal(0, 2.0, size=(B, 8)).astype(np.float32))
    H = O.solve_dlt(batch["pts1"], h4p).float()
    I = batch["I_aug"].numpy()
    ox, oy = batch["pts1"][:, 0].long().numpy(), batch["pts1"][:, 1].long().numpy()
    t = R.warp_window(I, H.numpy().reshape(B, 9), ox, oy, 128, 128)
    ref = O.transform(batch["I_aug"].double(), H.double(), batch["patch_indices"], 128).numpy()[..., 0]
    x64, y64 = _coords64(H.numpy(), 320, 240, ox, oy, 128, 128)
    dx, dy = np.abs(t["x"] - x64), np.abs(t["y"] - y64)
    # fp32 coordinates of ~300 px carry a few ulp of the H' entries and the divisions: well under 1e-3 px
    assert dx.max() < 1e-3 and dy.max() < 1e-3, (dx.max(), dy.max())
    same = (np.floor(t["x"]) == np.floor(x64)) & (np.floor(t["y"]) == np.floor(y64))
    assert same.mean() > 0.999
    slope = 2 * np.abs(I).max()                         # |d bilinear / dx| <= max |I_k - I_j|
    cond = R.blend_magnitude(I, t, np.arange(B)[:, None, None])
    err = np.abs(t["pv"] - ref)
    assert (err[same] <= slope * (dx + dy)[same] + 16 * R.U32 * cond[same] + 1e-12).all(), err[same].max()


def test_restated_full_transformer_matches_fp64():
    rng = np.random.default_rng(2)
    U = rng.normal(size=(2, 24, 32, 3)).astype(f32)
    theta = np.eye(3, dtype=f32)[None].repeat(2, 0)
    theta[1] = np.array([[0.9, 0.1, 0.05], [-0.08, 1.1, 0.0], [0.02, -0.03, 1.0]], f32)
    out = R.transformer(U, theta.reshape(2, 9), 24, 32)
    ref, _ = O.transformer(torch.tensor(U).double(), torch.tensor(theta).double(), (24, 32))
    assert np.abs(out - ref.numpy()).max() < 1e-4


def test_restated_dlt_system_bit_identical():
    rng = np.random.default_rng(3)
    B = 64
    x0 = rng.integers(45, 148, size=B); y0 = rng.integers(45, 68, size=B)
    pts1 = np.stack([x0, y0, x0 + 128, y0, x0 + 128, y0 + 128, x0, y0 + 128], 1).astype(f32)
    h4p = rng.uniform(-45, 45, size=(B, 8)).astype(f32)
    A, b = R.dlt_system(pts1, h4p)
    pts2 = torch.tensor((pts1 + h4p).astype(f32)).double()
    Ao, bo = O.dlt_system(torch.tensor(pts1).double(), pts2)
    assert np.array_equal(A, Ao.numpy()) and np.array_equal(b, bo.numpy()[..., 0])
    H, cond = R.dlt_fwd(pts1, h4p)
    Href = O.solve_dlt(torch.tensor(pts1).double(), pts2 - torch.tensor(pts1).double()).numpy().reshape(B, 9)
    assert np.abs(H - Href).max() <= 1e-9 * np.abs(Href).max() and (cond > 1e3).all()


def test_restated_backward_terms_match_autograd_of_the_restated_sampler():
    """bwd_terms is the derivative of the restated bilinear through x = (xs/ts + 1) W / 2: check it against fp64 autograd
    of the same map (gates frozen at the restated cells) for one L1-like upstream."""
    B = 2
    batch = O.make_batch(7, B)
    H = batch["H_gt"].float().numpy().reshape(B, 9)
    I = batch["I_aug"].numpy()
    ox, oy = batch["pts1"][:, 0].long().numpy(), batch["pts1"][:, 1].long().numpy()
    t = R.warp_window(I, H, ox, oy, 16, 8)
    gp = np.random.default_rng(0).normal(size=t["pv"].shape)
    terms, mag = R.bwd_terms(I, t, gp, np.abs(gp))
    # autograd: pv(H') with the restated cells frozen
    Hn = torch.tensor(t["Hn"].astype(np.float64), requires_grad=True)
    xt, yt = torch.tensor(t["xt"].astype(np.float64)), torch.tensor(t["yt"].astype(np.float64))
    h = Hn[:, None, None, :]
    ts = h[..., 6] * xt + h[..., 7] * yt + h[..., 8]
    x =((h[..., 0] * xt + h[..., 1] * yt + h[..., 2]) / ts + 1) * 160
    y = ((h[..., 3] * xt + h[..., 4] * yt + h[..., 5]) / ts + 1) * 120
    Ia, Ib, Ic, Id = [torch.tensor(g.astype(np.float64)) for g in R.gather(I, t, np.arange(B)[:, None, None])]
    f = lambda k: torch.tensor(t[k].astype(np.float64))[..., None]
    xx, yy = x[..., None], y[..., None]
    v = ((f("x1f") - xx) * (f("y1f") - yy) * Ia + (f("x1f") - xx) * (yy - f("y0f")) * Ib
         + (xx - f("x0f")) * (f("y1f") - yy) * Ic + (xx - f("x0f")) * (yy - f("y0f")) * Id).mean(-1)
    (v * torch.tensor(gp)).sum().backward()
    got = terms.sum(axis=(1, 2))
    # the terms use the fp32 xn, yn, ts, the autograd map their fp64 recomputation: a few fp32 ulp apart
    assert (np.abs(got - Hn.grad.numpy()) <= 1e-5 * mag.sum(axis=(1, 2))).all()
