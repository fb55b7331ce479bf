"""NumPy restatement of the photometric kernels' fp32 arithmetic — TEST INFRASTRUCTURE ONLY.

`csrc/warp.cu` builds every gate of the warp from plain fp32 operations: explicit `fmaf`, `__fmul_rn` / `__fadd_rn`, IEEE
division and `floorf` (the build has no fast-math).  This module repeats those operations in NumPy float32, line by line,
so that the sampler's coordinates, clipped cells, weights and gray values are reproduced bit for bit.  The one operation it
cannot repeat is the forward's `rcp.approx` (warp.cu `source_xy`); `forward_coord_delta` bounds its effect instead.

On top of the restated gates, the backward's per-pixel contributions (warp.cu `warp_loss_bwd_kernel`), the conjugation
`conj_bwd` and the DLT (csrc/dlt.cu) are evaluated in fp64, so that what is left between a kernel and this module is the
kernel's own fp32 summation rounding.  Line references are to csrc/warp.cu and csrc/dlt.cu.
"""
import numpy as np

f32 = np.float32
U32 = 2.0 ** -24           # unit roundoff of fp32
U64 = 2.0 ** -53


def fmaf32(a, b, c):
    """fmaf(a, b, c) on float32 arrays, exactly rounded (round to nearest even).

    The fp64 product of two fp32 values is exact; the fp64 sum s = p + c is not, and rounding s to fp32 rounds twice.
    That is wrong only when s lands exactly on an fp32 midpoint while the exact sum does not: the TwoSum residual e then
    says on which side of the midpoint the exact sum lies."""
    a = np.asarray(a, f32); b = np.asarray(b, f32); c = np.asarray(c, f32)
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        s = p + c64
        bb = s - p
        e = (p - (s - bb)) + (c64 - bb)                     # TwoSum: p + c = s + e exactly
        r = s.astype(f32)
        r64 = r.astype(np.float64)
        other = (2.0 * s - r64)                              # the other fp32 neighbour when s is a midpoint
        mid = (r64 != s) & (other.astype(f32).astype(np.float64) == other) & np.isfinite(s) & (e != 0)
        if np.any(mid):
            o32 = other.astype(f32)
            up = np.where(r64 > o32.astype(np.float64), r, o32)
            dn = np.where(r64 > o32.astype(np.float64), o32, r)
            r = np.where(mid, np.where(e > 0, up, dn), r)
    return r.astype(f32)


def normalise_h(Hp, img_w, img_h):
    """H' = (M^-1 . H) . M in the kernel's fp32 order (:21-39).  Hp [B,9] fp32 -> [B,9] fp32."""
    Hp = np.asarray(Hp, f32).reshape(-1, 9)
    sx, sy = f32(0.5) * f32(img_w), f32(0.5) * f32(img_h)
    ix, iy = f32(1) / sx, f32(1) / sy
    t = np.empty_like(Hp)
    for c in range(3):
        t[:, c] = fmaf32(ix, Hp[:, c], -Hp[:, 6 + c])
        t[:, 3 + c] = fmaf32(iy, Hp[:, 3 + c], -Hp[:, 6 + c])
        t[:, 6 + c] = Hp[:, 6 + c]
    o = np.empty_like(Hp)
    for r in range(3):
        o[:, 3 * r] = t[:, 3 * r] * sx
        o[:, 3 * r + 1] = t[:, 3 * r + 1] * sy
        o[:, 3 * r + 2] = fmaf32(t[:, 3 * r], sx, fmaf32(t[:, 3 * r + 1], sy, t[:, 3 * r + 2]))
    return o


def step(n):
    """TF LinSpace step 2 / (n - 1) in fp32 (:221-222)."""
    return f32(2) / f32(n - 1)


def grid_coord(stp, i):
    """fmaf(step, (float)i, -1) (:241, :246)."""
    return fmaf32(stp, np.asarray(i, f32), f32(-1))


def tap_from_xy(x, y, W, Hh):
    """Clip-then-weight taps (:49-66): dict of the int cell corners, their float copies and the four weights."""
    x = np.asarray(x, f32); y = np.asarray(y, f32)
    with np.errstate(invalid="ignore"):
        xf = np.fmin(np.fmax(np.floor(x), f32(-2)), f32(W) + f32(1))
        yf = np.fmin(np.fmax(np.floor(y), f32(-2)), f32(Hh) + f32(1))
    x0 = np.where(x == x, xf, 0).astype(np.int64)
    y0 = np.where(y == y, yf, 0).astype(np.int64)
    x1, y1 = x0 + 1, y0 + 1
    x0 = np.clip(x0, 0, W - 1); x1 = np.clip(x1, 0, W - 1)
    y0 = np.clip(y0, 0, Hh - 1); y1 = np.clip(y1, 0, Hh - 1)
    x0f, x1f, y0f, y1f = x0.astype(f32), x1.astype(f32), y0.astype(f32), y1.astype(f32)
    with np.errstate(invalid="ignore", over="ignore"):
        wa = (x1f - x) * (y1f - y)
        wb = (x1f - x) * (y - y0f)
        wc = (x - x0f) * (y1f - y)
        wd = (x - x0f) * (y - y0f)
    return dict(x=x, y=y, x0=x0, x1=x1, y0=y0, y1=y1, x0f=x0f, x1f=x1f, y0f=y0f, y1f=y1f, wa=wa, wb=wb, wc=wc, wd=wd)


def sample_setup(h, xt, yt, W, Hh):
    """Source coordinates of grid point (xt, yt) (:70-80).  h [..., 9] normalised H' broadcast against xt, yt."""
    h = [np.asarray(h[..., i], f32) for i in range(9)]
    xs = fmaf32(h[0], xt, fmaf32(h[1], yt, h[2]))
    ys = fmaf32(h[3], xt, fmaf32(h[4], yt, h[5]))
    ts = fmaf32(h[6], xt, fmaf32(h[7], yt, h[8]))
    ts = np.where(np.abs(ts) >= f32(1e-7), ts, ts + f32(1e-6)).astype(f32)   # smallers rule (:74)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        xn = xs / ts
        yn = ys / ts
        x = (xn + f32(1)) * f32(W) / f32(2)
        y = (yn + f32(1)) * f32(Hh) / f32(2)
    t = tap_from_xy(x, y, W, Hh)
    t.update(xs=xs, ys=ys, ts=ts, xn=xn, yn=yn)
    return t


def gather(img, t, b):
    """Ia, Ib, Ic, Id [..., C] fp32 of the taps; img [B,Hh,W,C], b the sample index broadcast against the taps."""
    b = np.broadcast_to(b, t["x0"].shape)
    return (img[b, t["y0"], t["x0"]], img[b, t["y1"], t["x0"]], img[b, t["y0"], t["x1"]], img[b, t["y1"], t["x1"]])


def bilinear_rn(t, Ia, Ib, Ic, Id):
    """((wa*Ia + wb*Ib) + wc*Ic) + wd*Id, every product and sum rounded (:85-87).  I* [..., C]; weights broadcast."""
    w = [t[k][..., None] for k in ("wa", "wb", "wc", "wd")]
    with np.errstate(invalid="ignore", over="ignore"):
        return ((w[0] * Ia + w[1] * Ib) + w[2] * Ic) + w[3] * Id


def sample_gray(img, t, b):
    """sample_gray<C> (:89-99): channel blends summed left to right from 0, divided by C when C = 3."""
    v = bilinear_rn(t, *gather(img, t, b))
    C = img.shape[-1]
    acc = np.zeros(v.shape[:-1], f32)
    for c in range(C):
        acc = acc + v[..., c]
    return acc if C == 1 else acc / f32(C)


def blend_magnitude(img, t, b):
    """sum_c sum_k |w_k I_k| / C: the scale of the rounding of a blend (the black border cancels at this scale)."""
    Ia, Ib, Ic, Id = gather(img, t, b)
    m = sum(np.abs(t[k][..., None].astype(np.float64) * I.astype(np.float64))
            for k, I in zip(("wa", "wb", "wc", "wd"), (Ia, Ib, Ic, Id)))
    return m.sum(-1) / img.shape[-1]


def window_grid(Hn, W, Hh, ox, oy, pw, ph):
    """xt [1,1,pw], yt [1,ph,1] grids of the windows at origins ox, oy [B] (window_origin, :116-123)."""
    sx, sy = step(W), step(Hh)
    cols = np.asarray(ox, np.int64)[:, None, None] + np.arange(pw)[None, None, :]
    rows = np.asarray(oy, np.int64)[:, None, None] + np.arange(ph)[None, :, None]
    return grid_coord(sx, cols), grid_coord(sy, rows)


def warp_window(I, H, ox, oy, pw, ph):
    """The backward's restated sampler on the windows: dict of per-pixel arrays [B,ph,pw] (pv = the gray value).
    I [B,Hh,W,C] fp32, H [B,9] pixel-unit fp32, ox, oy [B] window origins."""
    I = np.asarray(I, f32)
    B, Hh, W, _ = I.shape
    Hn = normalise_h(H, W, Hh)
    xt, yt = window_grid(Hn, W, Hh, ox, oy, pw, ph)
    t = sample_setup(Hn[:, None, None, :], xt, yt, W, Hh)
    bidx = np.arange(B)[:, None, None]
    t["pv"] = sample_gray(I, t, bidx)
    t["xt"] = np.broadcast_to(xt, t["pv"].shape)
    t["yt"] = np.broadcast_to(yt, t["pv"].shape)
    t["Hn"] = Hn
    return t


def transformer(U, theta, oh, ow):
    """transformer_kernel (:474-494): theta [B,9] already normalised, full output grid, every channel."""
    U = np.asarray(U, f32)
    B, Hh, W, C = U.shape
    xt = grid_coord(step(ow), np.arange(ow))[None, None, :]
    yt = grid_coord(step(oh), np.arange(oh))[None, :, None]
    t = sample_setup(np.asarray(theta, f32).reshape(B, 1, 1, 9), xt, yt, W, Hh)
    return bilinear_rn(t, *gather(U, t, np.arange(B)[:, None, None]))


def warp_image_u8(U, H):
    """warp_image_u8_kernel (:501-522): uint8 [B,Hh,W,3] warped with the pixel-unit H [B,9]; clamp to [0,255] (NaN -> 0,
    fmaxf's rule), then truncate."""
    U = np.asarray(U)
    B, Hh, W, C = U.shape
    Hn = normalise_h(H, W, Hh)
    xt = grid_coord(step(W), np.arange(W))[None, None, :]
    yt = grid_coord(step(Hh), np.arange(Hh))[None, :, None]
    t = sample_setup(Hn.reshape(B, 1, 1, 9), xt, yt, W, Hh)
    v = bilinear_rn(t, *[g.astype(f32) for g in gather(U, t, np.arange(B)[:, None, None])])
    return np.fmin(np.fmax(v, f32(0)), f32(255)).astype(np.uint8)


# ------------------------------------------------------------------------------------------------ backward on given gates
def bwd_terms(I, t, gp, gp_abs):
    """The nine per-pixel contributions to dH' of :324-353 in fp64, on the restated fp32 taps `t` (from warp_window) and
    a given d loss / d pred `gp` (fp64, [B,ph,pw]).  gp_abs bounds |gp|'s fp32 operands (for the rounding bound).
    Returns (terms [B,ph,pw,9], magnitude [B,ph,pw,9]): the magnitude is each term with every sum replaced by the sum of
    the absolute values of its operands, the scale at which the kernel's fp32 evaluation of the term rounds."""
    I = np.asarray(I, f32)
    B, Hh, W, C = I.shape
    d = lambda k: t[k].astype(np.float64)
    Ia, Ib, Ic, Id = [g.astype(np.float64) for g in gather(I, t, np.arange(B)[:, None, None])]
    y, x = d("y")[..., None], d("x")[..., None]
    p1, p2 = (d("y1f")[..., None] - y) * (Ic - Ia), (y - d("y0f")[..., None]) * (Id - Ib)
    q1, q2 = (d("x1f")[..., None] - x) * (Ib - Ia), (x - d("x0f")[..., None]) * (Id - Ic)
    gx, gy = (p1 + p2).sum(-1) / C, (q1 + q2).sum(-1) / C
    gxa, gya = (np.abs(p1) + np.abs(p2)).sum(-1) / C, (np.abs(q1) + np.abs(q2)).sum(-1) / C
    Gx, Gy = gp * gx * (0.5 * W), gp * gy * (0.5 * Hh)
    Gxa, Gya = gp_abs * gxa * (0.5 * W), gp_abs * gya * (0.5 * Hh)
    inv_t = 1.0 / d("ts")
    xn, yn, xt, yt = d("xn"), d("yn"), d("xt"), d("yt")
    dxs, dys = Gx * inv_t, Gy * inv_t
    dts = -(Gx * xn + Gy * yn) * inv_t
    dxa, dya = np.abs(Gxa * inv_t), np.abs(Gya * inv_t)
    dta = (np.abs(Gxa * xn) + np.abs(Gya * yn)) * np.abs(inv_t)
    terms = np.stack([dxs * xt, dxs * yt, dxs, dys * xt, dys * yt, dys, dts * xt, dts * yt, dts], -1)
    mag = np.stack([dxa * abs(xt), dxa * abs(yt), dxa, dya * abs(xt), dya * abs(yt), dya, dta * abs(xt), dta * abs(yt), dta], -1)
    return terms, mag


def conj_bwd(dHn, img_w, img_h):
    """dH = M^-T-style adjoint of H' = M^-1 H M (:363-385) in fp64 on the fp32 constants; also the magnitude of each
    element (sums of absolute operands).  dHn [B,9] -> ([B,9], [B,9])."""
    sx, sy = 0.5 * float(f32(img_w)), 0.5 * float(f32(img_h))
    ix, iy = float(f32(1) / f32(sx)), float(f32(1) / f32(sy))
    g = np.asarray(dHn, np.float64).reshape(-1, 9)
    out, mag = np.empty_like(g), np.empty_like(g)
    t, ta = np.empty_like(g), np.empty_like(g)
    for r in range(3):
        t[:, 3 * r] = sx * (g[:, 3 * r] + g[:, 3 * r + 2]); ta[:, 3 * r] = sx * (abs(g[:, 3 * r]) + abs(g[:, 3 * r + 2]))
        t[:, 3 * r + 1] = sy * (g[:, 3 * r + 1] + g[:, 3 * r + 2]); ta[:, 3 * r + 1] = sy * (abs(g[:, 3 * r + 1]) + abs(g[:, 3 * r + 2]))
        t[:, 3 * r + 2] = g[:, 3 * r + 2]; ta[:, 3 * r + 2] = abs(g[:, 3 * r + 2])
    for c in range(3):
        out[:, c] = ix * t[:, c]; mag[:, c] = ix * ta[:, c]
        out[:, 3 + c] = iy * t[:, 3 + c]; mag[:, 3 + c] = iy * ta[:, 3 + c]
        out[:, 6 + c] = t[:, 6 + c] - t[:, c] - t[:, 3 + c]; mag[:, 6 + c] = ta[:, 6 + c] + ta[:, c] + ta[:, 3 + c]
    return out, mag


def forward_coord_delta(t, W, Hh):
    """Bound on |x_f - x_b| and |y_f - y_b| between the forward's coordinates (one rcp.approx, <= 1 ulp by the PTX ISA,
    then xs * rt + 1 fused or not, * W, * 0.5) and the restated IEEE ones (xs / ts, + 1, * W, / 2)."""
    xn, yn = np.abs(t["xn"].astype(np.float64)), np.abs(t["yn"].astype(np.float64))
    dx = 0.5 * W * (xn * 2.0 ** -22 + 4 * U32 * (xn + 1.0))
    dy = 0.5 * Hh * (yn * 2.0 ** -22 + 4 * U32 * (yn + 1.0))
    return dx * 1.01, dy * 1.01


def box_candidates(v, dv):
    """fp32 abscissae at which the restated bilinear can take its extremes over [v - dv, v + dv]: the box ends and, for
    each integer (cell or clip boundary) inside the box, the integer and the fp32 number just below it.  [..., 4]."""
    v64 = v.astype(np.float64)
    lo, hi = (v64 - dv).astype(f32), (v64 + dv).astype(f32)
    k = np.floor(hi.astype(np.float64))
    inside = (k > lo.astype(np.float64)) & np.isfinite(k)
    kk = np.where(inside, k, v64).astype(f32)
    below = np.where(inside, np.nextafter(kk, f32(-np.inf)), v)
    return np.stack([lo, hi, kk, below], -1)


# ------------------------------------------------------------------------------------------------ DLT (csrc/dlt.cu)
def dlt_system(pts1, h4p):
    """A [B,8,8], b [B,8] in fp64 as build_row (dlt.cu:49-58) builds them: pts2 = pts1 + h4p rounded to fp32 first."""
    p1 = np.asarray(pts1, f32).reshape(-1, 4, 2)
    p2 = (p1 + np.asarray(h4p, f32).reshape(-1, 4, 2)).astype(f32)
    x, y = p1[..., 0].astype(np.float64), p1[..., 1].astype(np.float64)
    u, v = p2[..., 0].astype(np.float64), p2[..., 1].astype(np.float64)
    z, o = np.zeros_like(x), np.ones_like(x)
    r0 = np.stack([z, z, z, -x, -y, -o, v * x, v * y], -1)
    r1 = np.stack([x, y, o, z, z, z, -u * x, -u * y], -1)
    A = np.stack([r0, r1], 2).reshape(-1, 8, 8)
    b = np.stack([-v, u], 2).reshape(-1, 8)
    return A, b


def dlt_fwd(pts1, h4p):
    """(H [B,9] fp64 with h33 = 1, cond_2(A) [B])."""
    A, b = dlt_system(pts1, h4p)
    h = np.linalg.solve(A, b[..., None])[..., 0]
    return np.concatenate([h, np.ones((h.shape[0], 1))], 1), np.linalg.cond(A)


def dlt_bwd(pts1, h4p, H, dH):
    """dh4p [B,8] in fp64 (dlt.cu:79-124): lambda = A^-T dH[0:8], s_i = h6 x_i + h7 y_i + 1 from the given fp32 H.
    Also returns max|lambda * s| per sample and cond_2(A)."""
    A, _ = dlt_system(pts1, h4p)
    lam = np.linalg.solve(np.transpose(A, (0, 2, 1)), np.asarray(dH, np.float64).reshape(-1, 9)[:, :8, None])[..., 0]
    p1 = np.asarray(pts1, f32).reshape(-1, 4, 2).astype(np.float64)
    Hd = np.asarray(H, f32).reshape(-1, 9).astype(np.float64)
    s = Hd[:, 6:7] * p1[..., 0] + Hd[:, 7:8] * p1[..., 1] + 1.0
    out = np.empty((A.shape[0], 8))
    out[:, 0::2] = lam[:, 1::2] * s
    out[:, 1::2] = -lam[:, 0::2] * s
    scale = np.abs(lam).max(1) * np.abs(s).max(1)
    return out, scale, np.linalg.cond(A)
