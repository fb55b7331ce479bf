"""The mosaic's multi-band blend (udh_mosaic_multiband_u8, bit for bit): cv2.detail_MultiBandBlender with CV_16S weights,
fed each frame's warp on its own ROI of the canvas (test infrastructure only).

Inputs: kept frames F_k uint8 RGB [h_k,w_k,3], float64 M_k (frame k -> canvas, as mosaic.canvas returns them), a canvas
Hc x Wc and B bands.
  ROI       mosaic.multiband_rois: the frame's mapped pixel-centre corners give x_lo = max(0, floor(min x) - 1), x_hi =
            min(Wc, ceil(max x) + 2) (exclusive), likewise in y; tl_k = (x_lo, y_lo), M'_k = T(-tl_k) M_k in float64.
  fed       img_k = cv2.warpPerspective(F_k, M'_k, (x_hi - x_lo, y_hi - y_lo)); mask_k = 255 where
            oracle/mosaic.validity_weight(M'_k, h_k, w_k, roi_h, roi_w, 0) finds the pixel valid, else 0.
  blend     cv2.ocl.setUseOpenCL(False); b = cv2.detail_MultiBandBlender(0, B, cv2.CV_16S); b.prepare((0, 0, Wc, Hc));
            b.feed(img_k, mask_k, tl_k) per frame; dst, dst_mask = b.blend(None, None); mosaic = saturate_u8(dst).

restate() states cv2's integer rule in NumPy (every point is checked against cv2 by tests/test_multiband_logic.py):
  bands     B' = min(B, ceil(log(max(Wc, Hc)) / log(2))) in float64; the canvas is padded up to multiples of 2^B'.
  rectangle a frame's rectangle is its ROI grown by the gap 3 2^B' on each side, clipped to the padded canvas, its
            top-left floored to a multiple of 2^B', its size rounded up to one, then shifted left / up by what passes the
            padded canvas's far edge (cv2's tl_new / br_new).  At level i it is the rectangle's coordinates >> i.
  image     the ROI warp bordered with BORDER_REFLECT (folding as often as the border needs); G_0 = that, G_{i+1} =
            pyr_down(G_i) in uint8; L_i = G_i - pyr_up(G_{i+1}) in int16, L_B' = G_B'.
  weight    mask -> int16, + 1 where nonzero (255 -> 256), bordered with a constant 0; W_{i+1} = pyr_down(W_i) in int16.
  feed      acc_i += (int16)((L_i W_i) >> 8) and wacc_i += W_i over the rectangle: wrapping int16 adds.
  blend     N_i = (int16)((acc_i << 8) / (wacc_i + 1)) (C division, truncating); R_B' = N_B', R_i = sat16(pyr_up(R_{i+1})
            + N_i); crop to Hc x Wc; mask = wacc_0 > 0 (signed); dst = R_0 where mask else 0; mosaic = saturate_u8(dst).
  pyramids  pyr_down: taps 1 4 6 4 1 at 2x - 2 .. 2x + 2 with BORDER_REFLECT_101, (sum + 128) >> 8, size (n + 1) // 2.
            pyr_up: output 2j = s[j-1] + 6 s[j] + s[j+1], 2j + 1 = 4 s[j] + 4 s[j+1], (sum + 32) >> 6 over both axes,
            saturated; index -1 reads s[1] (s[0] when n = 1) but index n reads s[n-1]: reflect-101 on the left and top,
            reflect on the right and bottom.
The normalisation divides by wacc + 1, so a lone frame of 255 comes out 254: that is cv2's result, kept.
"""
import math

import numpy as np

from . import mosaic as OM


# ---- pyramids --------------------------------------------------------------------------------------------------------------
def reflect101(i, n):
    i = np.asarray(i, np.int64)
    if n == 1:
        return np.zeros_like(i)
    p = np.abs(i) % (2 * n - 2)
    return np.where(p >= n, 2 * n - 2 - p, p)


def reflect(i, n):
    """BORDER_REFLECT (fedcba|abcdef|fedcba), folding as often as needed."""
    i = np.asarray(i, np.int64)
    if n == 1:
        return np.zeros_like(i)
    p = i % (2 * n)
    return np.where(p >= n, 2 * n - 1 - p, p)


def _limits(dtype):
    info = np.iinfo(dtype)
    return info.min, info.max


def pyr_down(a):
    """cv2.pyrDown of a uint8 or int16 [H,W] or [H,W,C] array."""
    a = np.asarray(a)
    H, W = a.shape[:2]
    k = (1, 4, 6, 4, 1)
    x = 2 * np.arange((W + 1) // 2)
    t = sum(kk * a[:, reflect101(x + j - 2, W)].astype(np.int64) for j, kk in enumerate(k))
    y = 2 * np.arange((H + 1) // 2)
    t = sum(kk * t[reflect101(y + j - 2, H)] for j, kk in enumerate(k))
    return np.clip((t + 128) >> 8, *_limits(a.dtype)).astype(a.dtype)


def _up_taps(n):
    """-> (index [2n,3], weight [2n,3]) of pyr_up along one axis of length n."""
    j = np.arange(n)
    idx = np.zeros((2 * n, 3), np.int64)
    wt = np.zeros((2 * n, 3), np.int64)
    idx[0::2] = np.stack([j - 1, j, j + 1], 1)
    wt[0::2] = (1, 6, 1)
    idx[1::2] = np.stack([j, j + 1, j + 1], 1)
    wt[1::2] = (4, 4, 0)
    idx = np.where(idx < 0, min(1, n - 1), idx)
    return np.minimum(idx, n - 1), wt


def pyr_up(a):
    """cv2.pyrUp of a uint8 or int16 [H,W] or [H,W,C] array (to 2H x 2W)."""
    a = np.asarray(a)
    H, W = a.shape[:2]
    ix, wx = _up_taps(W)
    iy, wy = _up_taps(H)
    t = sum(wx[:, j].reshape((1, -1) + (1,) * (a.ndim - 2)) * a[:, ix[:, j]].astype(np.int64) for j in range(3))
    t = sum(wy[:, j].reshape((-1,) + (1,) * (a.ndim - 1)) * t[iy[:, j]] for j in range(3))
    return np.clip((t + 32) >> 6, *_limits(a.dtype)).astype(a.dtype)


# ---- the rectangles --------------------------------------------------------------------------------------------------------
def num_bands(Hc, Wc, bands):
    return min(int(bands), int(math.ceil(math.log(float(max(Wc, Hc))) / math.log(2.0))))


def padded_rect(tx, ty, roi_w, roi_h, Hp, Wp, B):
    """cv2's fed rectangle (x0, y0, x1, y1) at level 0 of an roi_h x roi_w image at (tx, ty) on the padded canvas."""
    gap, a = 3 << B, 1 << B
    x0, y0 = max(0, tx - gap), max(0, ty - gap)
    x1, y1 = min(Wp, tx + roi_w + gap), min(Hp, ty + roi_h + gap)
    x0, y0 = (x0 >> B) << B, (y0 >> B) << B
    w, h = x1 - x0, y1 - y0
    x1, y1 = x0 + w + (a - w % a) % a, y0 + h + (a - h % a) % a
    dx, dy = max(x1 - Wp, 0), max(y1 - Hp, 0)
    return x0 - dx, y0 - dy, x1 - dx, y1 - dy


def level_pyramids(img, mask, tl, Hp, Wp, B):
    """One fed frame -> (rect, L [B+1] int16 [h_i,w_i,3], W [B+1] int16 [h_i,w_i])."""
    rh, rw = mask.shape
    tx, ty = tl
    x0, y0, x1, y1 = padded_rect(tx, ty, rw, rh, Hp, Wp, B)
    ys, xs = np.arange(y0, y1) - ty, np.arange(x0, x1) - tx
    g = img[reflect(ys, rh)][:, reflect(xs, rw)]
    wm = np.where(mask != 0, mask.astype(np.int16) + 1, 0).astype(np.int16)
    inside = ((ys >= 0) & (ys < rh))[:, None] & ((xs >= 0) & (xs < rw))[None, :]
    w0 = np.zeros(inside.shape, np.int16)
    w0[inside] = wm[ys[(ys >= 0) & (ys < rh)]][:, xs[(xs >= 0) & (xs < rw)]].ravel()
    G, W = [g], [w0]
    for _ in range(B):
        G.append(pyr_down(G[-1]))
        W.append(pyr_down(W[-1]))
    L = [(G[i].astype(np.int16) - pyr_up(G[i + 1]).astype(np.int16)).astype(np.int16) for i in range(B)] + [G[B].astype(np.int16)]
    return (x0, y0, x1, y1), L, W


def restate(imgs, masks, tls, Hc, Wc, bands):
    """Fed images (uint8 [h,w,3]), masks (uint8 [h,w]) and top-lefts (x, y) -> dict(mosaic uint8 [Hc,Wc,3], mask uint8
    [Hc,Wc], dst int16 [Hc,Wc,3], bands B', acc [B'+1] int16 [Hp>>i,Wp>>i,3], wacc [B'+1] int16 [Hp>>i,Wp>>i]): cv2's
    integer rule, with each level's sums as they stand before the blend normalises them."""
    B = num_bands(Hc, Wc, bands)
    a = 1 << B
    Hp, Wp = Hc + (-Hc) % a, Wc + (-Wc) % a
    acc = [np.zeros((Hp >> i, Wp >> i, 3), np.int16) for i in range(B + 1)]
    wacc = [np.zeros((Hp >> i, Wp >> i), np.int16) for i in range(B + 1)]
    for img, mask, tl in zip(imgs, masks, tls):
        (x0, y0, x1, y1), L, W = level_pyramids(img, mask, tl, Hp, Wp, B)
        for i in range(B + 1):
            sl = (slice(y0 >> i, y1 >> i), slice(x0 >> i, x1 >> i))
            acc[i][sl] += ((L[i].astype(np.int32) * W[i][..., None]) >> 8).astype(np.int16)
            wacc[i][sl] += W[i]
    R = None
    for i in range(B, -1, -1):
        w = wacc[i].astype(np.int64)[..., None] + 1
        if (w == 0).any():
            raise ZeroDivisionError("level %d: a weight sum of -1 (cv2 divides by zero there)" % i)
        v = acc[i].astype(np.int64) << 8
        N = (np.sign(v) * np.sign(w) * (np.abs(v) // np.abs(w))).astype(np.int16)
        R = N if R is None else np.clip(pyr_up(R).astype(np.int32) + N, -32768, 32767).astype(np.int16)
    m = wacc[0][:Hc, :Wc] > 0
    dst = np.where(m[..., None], R[:Hc, :Wc], 0).astype(np.int16)
    return dict(mosaic=np.clip(dst, 0, 255).astype(np.uint8), mask=np.where(m, 255, 0).astype(np.uint8), dst=dst, bands=B,
                acc=acc, wacc=wacc)


# ---- cv2 --------------------------------------------------------------------------------------------------------------------
def fed(frames, M, Hc, Wc):
    """Kept frames and their M (frame -> canvas) -> (imgs, masks, tls) as the blender is fed; a frame whose ROI is empty
    (it misses the canvas) is left out."""
    import cv2
    from unsuperviseddeephomographyral2018_b200 import mosaic
    rois, Mr = mosaic.multiband_rois(M, [f.shape[:2] for f in frames], Hc, Wc)
    imgs, masks, tls = [], [], []
    for F, (x0, y0, x1, y1), Mk in zip(frames, rois, Mr):
        if x1 <= x0 or y1 <= y0:
            continue
        h, w = F.shape[:2]
        imgs.append(cv2.warpPerspective(F, Mk, (int(x1 - x0), int(y1 - y0))))
        valid, _ = OM.validity_weight(Mk, h, w, int(y1 - y0), int(x1 - x0), 0)
        masks.append(np.where(valid, 255, 0).astype(np.uint8))
        tls.append((int(x0), int(y0)))
    return imgs, masks, tls


def cv2_blend(imgs, masks, tls, Hc, Wc, bands):
    """cv2.detail_MultiBandBlender (CPU, CV_16S weights) -> (mosaic uint8 [Hc,Wc,3], mask uint8 [Hc,Wc], dst int16)."""
    import cv2
    cv2.ocl.setUseOpenCL(False)
    b = cv2.detail_MultiBandBlender(0, int(bands), cv2.CV_16S)
    b.prepare((0, 0, int(Wc), int(Hc)))
    for img, mask, tl in zip(imgs, masks, tls):
        b.feed(img, mask, (int(tl[0]), int(tl[1])))
    dst, dst_mask = b.blend(None, None)
    return np.clip(dst, 0, 255).astype(np.uint8), dst_mask, dst


def blend(frames, M, Hc, Wc, bands):
    """frames: uint8 RGB [h_k,w_k,3], M [n,3,3] (frame k -> canvas) -> (mosaic uint8 [Hc,Wc,3], mask uint8 [Hc,Wc])."""
    imgs, masks, tls = fed(frames, np.asarray(M, np.float64).reshape(-1, 3, 3), Hc, Wc)
    out, mask, _ = cv2_blend(imgs, masks, tls, Hc, Wc, bands)
    return out, mask
