"""The mosaic blend rule, restated with cv2 and NumPy (test infrastructure only); udh_mosaic_blend_u8 computes it bit for bit.

Inputs: frames F_k uint8 [h_k,w_k,C] (C = 1 or 3), float64 M_k (frame k -> canvas), a canvas Hc x Wc and an integer
feather >= 0 in source pixels.  For each canvas pixel and frame k:
  position  (X, Y), the frame's source position in 1/32 px exactly as cv2.warpPerspective(F_k, M_k, (Wc, Hc)) computes it
            (oracle/warp_perspective.source_coords: the canvas size's tile columns, the zero-denominator case); W is the
            denominator before 32 / W;
  valid     W != 0, 0 <= X <= 32 (w_k - 1) and 0 <= Y <= 32 (h_k - 1) (every tap with a nonzero weight is inside);
  value     v_k = that warpPerspective output value;
  weight    d = min(X, 32 (w_k - 1) - X, Y, 32 (h_k - 1) - Y), wt_k = 1 + min(d, 32 feather), all integer (feather = 0:
            a plain average).
Per channel S = sum wt_k v_k and D = sum wt_k over the valid frames in int64; out = (S + (D >> 1)) // D, mask = 255; where
D = 0, out = 0 and mask = 0.  The sums are integers, so the result depends neither on the frames' order nor on tiling.
Every frame is evaluated at every pixel: no candidate lists.
"""
import numpy as np

from . import warp_perspective as WP


def denominator(M, dst_h, dst_w):
    """float64 [dst_h, dst_w]: the W of source_coords before 32 / W (same operations, same order)."""
    Mi = WP.invert(M).reshape(-1)
    bw = WP.tile_width(dst_h, dst_w)
    x = np.arange(dst_w, dtype=np.float64)[None, :]
    y = np.arange(dst_h, dtype=np.float64)[:, None]
    xb = np.floor(x / bw) * bw
    return (Mi[6] * xb + Mi[7] * y + Mi[8]) + Mi[6] * (x - xb)


def validity_weight(M, h, w, dst_h, dst_w, feather):
    """-> (valid bool [dst_h,dst_w], wt int64 [dst_h,dst_w], 0 where invalid) of an h x w frame."""
    X, Y = WP.source_coords(M, dst_h, dst_w)
    xm, ym = 32 * (w - 1), 32 * (h - 1)
    valid = (denominator(M, dst_h, dst_w) != 0) & (X >= 0) & (X <= xm) & (Y >= 0) & (Y <= ym)
    d = np.minimum(np.minimum(X, xm - X), np.minimum(Y, ym - Y))
    wt = np.where(valid, 1 + np.minimum(d, 32 * int(feather)), 0)
    return valid, wt


def blend(frames, M, dst_h, dst_w, feather):
    """frames: uint8 [h_k,w_k,C] arrays, M [n,3,3] -> (mosaic uint8 [dst_h,dst_w,C], mask uint8 [dst_h,dst_w])."""
    import cv2
    C = frames[0].shape[2] if frames[0].ndim == 3 else 1
    S = np.zeros((dst_h, dst_w, C), np.int64)
    D = np.zeros((dst_h, dst_w), np.int64)
    for F, Mk in zip(frames, np.asarray(M, np.float64).reshape(-1, 3, 3)):
        h, w = F.shape[:2]
        v = cv2.warpPerspective(F if C == 3 else F.reshape(h, w), Mk, (dst_w, dst_h)).reshape(dst_h, dst_w, C).astype(np.int64)
        _, wt = validity_weight(Mk, h, w, dst_h, dst_w, feather)
        S += wt[..., None] * v
        D += wt
    out = np.where(D[..., None] > 0, (S + (D >> 1)[..., None]) // np.maximum(D, 1)[..., None], 0).astype(np.uint8)
    return out, np.where(D > 0, 255, 0).astype(np.uint8)
