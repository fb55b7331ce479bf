"""NumPy restatement of the real-data loader's host arithmetic (test infrastructure only, like oracle/jpeg.py).

The real-data loader (code/dataloader.py:146-200) reads full-size images, augments and normalises them there, then
AREA-resizes them to the network size; images stored at the network size are first brought up to the full size.  On the
host these are two cv2.resize(INTER_AREA) calls, restated here in the order OpenCV evaluates them, plus the photometric
augmentation as a per-value table:

  resize_area_down_f32  fp32 downscale with a non-integer ratio on at least one axis: OpenCV's generic resizeArea
                        (imgproc/src/resize.cpp: computeResizeAreaTab + ResizeArea_Invoker).  For every source row of an
                        output row, buf[dx] is a sequential fp32 sum of S[sx] * alpha, from 0 and in table order; the
                        output is the sequential fp32 sum of beta * buf over those rows, the first term assigned.  No FMA.
  resize_area_up_u8     uint8 upscale: INTER_AREA turns into linear interpolation with area coefficients (resize.cpp,
                        `area_mode` in the coefficient setup), 11-bit fixed point (INTER_RESIZE_COEF_BITS); the vertical
                        pass is VResizeLinearVec_32s8u's ((b0*(r0>>4))>>16) + ((b1*(r1>>4))>>16) + 2) >> 2.
  value_table           (clip(v ** f32(g) * f32(br) * c, 0, 255) - mean) / std on v = 0..255: every step of the host
                        path is elementwise in the uint8 value and the channel, so looking the table up gives the host
                        path's values bit for bit.
  draw_tables           the per-sample tables and the [B,11] augmentation table, drawing from the loader's RNG in the
                        order _disk_batch_extended_host draws.
"""
import math

import numpy as np

MEAN_I = np.array([118.93, 113.97, 102.60], np.float32)
STD_I = np.array([69.85, 68.81, 72.45], np.float32)


# ---- fp32 INTER_AREA downscale ------------------------------------------------------------------------------------------
def area_tab(ssize, dsize):
    """computeResizeAreaTab (cn = 1): [(di, si, alpha)] with the weights computed in double and cast to float."""
    scale = 1.0 / (float(dsize) / float(ssize))
    tab = []
    for dx in range(dsize):
        fsx1 = dx * scale
        fsx2 = fsx1 + scale
        cell = min(scale, ssize - fsx1)
        sx1, sx2 = int(math.ceil(fsx1)), int(math.floor(fsx2))
        sx2 = min(sx2, ssize - 1)
        sx1 = min(sx1, sx2)
        if sx1 - fsx1 > 1e-3:
            tab.append((dx, sx1 - 1, np.float32((sx1 - fsx1) / cell)))
        for sx in range(sx1, sx2):
            tab.append((dx, sx, np.float32(1.0 / cell)))
        if fsx2 - sx2 > 1e-3:
            tab.append((dx, sx2, np.float32(min(min(fsx2 - sx2, 1.0), cell) / cell)))
    return tab


def area_is_generic(sh, sw, dh, dw):
    """True when cv2.resize(INTER_AREA) takes the generic resizeArea path: a downscale on both axes (scale >= 1) whose
    ratios are not both integers (integer ratios take resizeAreaFast, another summation order)."""
    if dh > sh or dw > sw:
        return False
    sx, sy = sw / dw, sh / dh
    return not (abs(sx - round(sx)) < np.finfo(np.float64).eps and abs(sy - round(sy)) < np.finfo(np.float64).eps)


def resize_area_down_f32(src, dh, dw):
    """cv2.resize(src, (dw, dh), interpolation=INTER_AREA) for fp32 [sh, sw, cn] on the generic path."""
    src = np.asarray(src, np.float32)
    sh, sw, cn = src.shape
    assert area_is_generic(sh, sw, dh, dw)
    buf = np.zeros((sh, dw, cn), np.float32)                       # the horizontal pass of every source row
    for dx, sx, a in area_tab(sw, dw):
        buf[:, dx] = buf[:, dx] + src[:, sx] * a
    out = np.empty((dh, dw, cn), np.float32)
    first = [True] * dh
    for dy, sy, beta in area_tab(sh, dh):
        if first[dy]:
            out[dy] = beta * buf[sy]
            first[dy] = False
        else:
            out[dy] = out[dy] + beta * buf[sy]
    return out


# ---- uint8 INTER_AREA upscale -------------------------------------------------------------------------------------------
def linear_area_coefs(ssize, dsize):
    """Per output index: first source index and the two 11-bit coefficients (cvRound(c * 2048)).  fx = (dx+1) -
    (sx+1) * inv_scale, then fx - floor(fx), in float; at the right border both taps sit on the last pixel."""
    inv = float(dsize) / float(ssize)
    scale = 1.0 / inv
    sx = np.empty(dsize, np.int64)
    a = np.empty((dsize, 2), np.int64)
    for dx in range(dsize):
        s = int(math.floor(dx * scale))
        fx = np.float32((dx + 1) - (s + 1) * inv)
        fx = np.float32(0) if fx <= 0 else np.float32(fx - math.floor(fx))
        c0, c1 = np.float32(1) - fx, fx
        if s >= ssize - 1:
            s, c0, c1 = ssize - 1, np.float32(1), np.float32(0)
        sx[dx] = s
        a[dx] = [int(np.rint(np.float32(c0 * np.float32(2048)))), int(np.rint(np.float32(c1 * np.float32(2048))))]
    return sx, a


def resize_area_up_u8(src, dh, dw):
    """cv2.resize(src, (dw, dh), interpolation=INTER_AREA) for uint8 [sh, sw, cn] with dh > sh and dw > sw."""
    src = np.asarray(src, np.uint8)
    sh, sw, cn = src.shape
    assert dh > sh and dw > sw
    sx, ax = linear_area_coefs(sw, dw)
    sy, ay = linear_area_coefs(sh, dh)
    S = src.astype(np.int64)
    nx = np.minimum(sx + 1, sw - 1)
    rows = S[:, sx] * ax[:, 0][None, :, None] + S[:, nx] * ax[:, 1][None, :, None]          # [sh, dw, cn]
    r0, r1 = rows[sy], rows[np.minimum(sy + 1, sh - 1)]
    b0, b1 = ay[:, 0][:, None, None], ay[:, 1][:, None, None]
    out = (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


# ---- augmentation + normalisation as a per-value table ------------------------------------------------------------------
def value_table(g=None, br=None, c=None):
    """[256, 3] fp32: the host path's augment (when g is not None) and normalise, evaluated on v = 0..255."""
    v = np.repeat(np.arange(256, dtype=np.float32)[:, None], 3, axis=1)
    if g is not None:
        v = np.clip(v ** np.float32(g) * np.float32(br) * c, 0, 255)
    return (v - MEAN_I) / STD_I


def draw_tables(rng, B, do_augment, mode):
    """-> (tables [B, 4, 256, 3] fp32 = plain I, plain I', augmented I, augmented I'; aug [B, 11] fp32 in
    udh_ecc_prep_u8's layout {on, gamma, brightness, colour RGB of I, the same five of I'}, zero when not augmented).
    Per sample: uniform(0, 1); when augmenting (g, br, c[3]); in test mode a second (g, br, c[3]) for I'."""
    plain = value_table()
    tables = np.empty((B, 4, 256, 3), np.float32)
    aug = np.zeros((B, 11), np.float32)
    for j in range(B):
        tables[j, 0] = tables[j, 1] = tables[j, 2] = tables[j, 3] = plain
        if rng.uniform(0, 1) > (1 - do_augment):
            draw = lambda: (rng.uniform(0.8, 1.2), rng.uniform(0.5, 2.0), rng.uniform(0.8, 1.2, size=3).astype(np.float32))
            a = draw()
            b = a if mode == 'train' else draw()
            tables[j, 2], tables[j, 3] = value_table(*a), value_table(*b)
            aug[j, 0] = 1.0
            aug[j, 1:6] = [a[0], a[1], *a[2]]
            aug[j, 6:11] = [b[0], b[1], *b[2]]
    return tables, aug
