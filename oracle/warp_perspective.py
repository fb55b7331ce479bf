"""NumPy restatement of cv2.warpPerspective(src, M, (dst_w, dst_h)) with its defaults (INTER_LINEAR, BORDER_CONSTANT,
border value 0) on uint8 images, as udh_warp_perspective_u8 computes it (test infrastructure only).  Each rule below was
settled by comparing against cv2.warpPerspective (tests/test_warp_perspective_oracle.py).

  inverse   M is inverted in float64 by the 3x3 cofactor rule: d = det (cofactor expansion along row 0), each inverse
            entry (a*b - c*e) * (1 / d); a singular M (d == 0) becomes the zero matrix.
  tiles     the output is walked in tiles of bh x bw pixels, bh = min(16, dst_h), bw = min(1024 // bh, dst_w); a pixel at
            column x of tile column xb = x - x % bw, row y:
              X0 = Mi[0] xb + Mi[1] y + Mi[2],  Y0 = Mi[3] xb + Mi[4] y + Mi[5],  W0 = Mi[6] xb + Mi[7] y + Mi[8]
              W  = W0 + Mi[6] (x - xb);  W = 32 / W, or 0 when W == 0
              X  = round_half_even(clamp((X0 + Mi[0] (x - xb)) W, INT_MIN, INT_MAX)), Y likewise
            every operation in float64, left to right, no fused multiply-add.  A zero denominator therefore lands on
            source pixel (0, 0).
  sample    source pixel (X >> 5, Y >> 5) (arithmetic shift, saturated to int16), fraction fx = X & 31, fy = Y & 31;
            weights 32 (32 - fx)(32 - fy), 32 fx (32 - fy), 32 (32 - fx) fy, 32 fx fy on the taps (sx, sy), (sx + 1, sy),
            (sx, sy + 1), (sx + 1, sy + 1); a tap outside the source contributes 0; out = (sum + 2^14) >> 15.
"""
import numpy as np

INT_MIN, INT_MAX = -2147483648.0, 2147483647.0


def invert(M):
    """cv2's float64 inverse of a 3x3 matrix (zero when singular), the one warpPerspective applies to M."""
    m = [[float(v) for v in row] for row in np.asarray(M, np.float64).reshape(3, 3)]
    d = (m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0])
         + m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]))
    if d == 0:
        return np.zeros((3, 3))
    d = 1.0 / d
    t = [(m[1][1] * m[2][2] - m[1][2] * m[2][1]) * d, (m[0][2] * m[2][1] - m[0][1] * m[2][2]) * d,
         (m[0][1] * m[1][2] - m[0][2] * m[1][1]) * d, (m[1][2] * m[2][0] - m[1][0] * m[2][2]) * d,
         (m[0][0] * m[2][2] - m[0][2] * m[2][0]) * d, (m[0][2] * m[1][0] - m[0][0] * m[1][2]) * d,
         (m[1][0] * m[2][1] - m[1][1] * m[2][0]) * d, (m[0][1] * m[2][0] - m[0][0] * m[2][1]) * d,
         (m[0][0] * m[1][1] - m[0][1] * m[1][0]) * d]
    return np.array(t).reshape(3, 3)


def tile_width(dst_h, dst_w):
    bh = min(16, dst_h)
    return min(1024 // bh, dst_w)


def source_coords(M, dst_h, dst_w):
    """-> (X, Y) int64 [dst_h, dst_w]: each output pixel's source position in 1/32 pixel."""
    Mi = invert(M).reshape(-1)
    bw = tile_width(dst_h, dst_w)
    x = np.arange(dst_w, dtype=np.float64)[None, :]
    y = np.arange(dst_h, dtype=np.float64)[:, None]
    xb = np.floor(x / bw) * bw
    x1 = x - xb
    X0 = Mi[0] * xb + Mi[1] * y + Mi[2]
    Y0 = Mi[3] * xb + Mi[4] * y + Mi[5]
    W0 = Mi[6] * xb + Mi[7] * y + Mi[8]
    W = W0 + Mi[6] * x1
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        W = np.where(W != 0, 32.0 / np.where(W != 0, W, 1.0), 0.0)
        fX = np.maximum(INT_MIN, np.minimum(INT_MAX, (X0 + Mi[0] * x1) * W))
        fY = np.maximum(INT_MIN, np.minimum(INT_MAX, (Y0 + Mi[3] * x1) * W))
    return np.rint(fX).astype(np.int64), np.rint(fY).astype(np.int64)


def warp_perspective(src, M, dsize):
    """uint8 [h,w] or [h,w,C], float64 M [3,3], dsize = (dst_w, dst_h) -> uint8 [dst_h,dst_w(,C)], equal to
    cv2.warpPerspective(src, M, dsize)."""
    dst_w, dst_h = dsize
    h, w = src.shape[:2]
    im = src.reshape(h, w, -1).astype(np.int64)
    X, Y = source_coords(M, dst_h, dst_w)
    sx, sy = np.clip(X >> 5, -32768, 32767), np.clip(Y >> 5, -32768, 32767)
    fx, fy = X & 31, Y & 31
    acc = np.zeros((dst_h, dst_w, im.shape[2]), np.int64)
    for dy, dx, wt in ((0, 0, (32 - fx) * (32 - fy)), (0, 1, fx * (32 - fy)), (1, 0, (32 - fx) * fy), (1, 1, fx * fy)):
        tx, ty = sx + dx, sy + dy
        inside = (tx >= 0) & (tx < w) & (ty >= 0) & (ty < h)
        v = im[np.clip(ty, 0, h - 1), np.clip(tx, 0, w - 1)] * inside[..., None]
        acc += v * (32 * wt)[..., None]
    out = ((acc + (1 << 14)) >> 15).astype(np.uint8)
    return out.reshape((dst_h, dst_w) + src.shape[2:])
