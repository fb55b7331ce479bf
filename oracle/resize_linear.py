"""NumPy restatement of cv2.resize(uint8, INTER_LINEAR) as udh_resize_linear_u8 computes it (test infrastructure only).

OpenCV's fixed-point path (resizeGeneric_): per axis f = (float)((d + 0.5) * scale - 0.5), s = floor(f), f -= s (float),
coefficients cvRound((1 - f) * 2048), cvRound(f * 2048) in float.  Columns at the borders: s < 0 -> (0, f = 0),
s >= size - 1 -> (size - 1, f = 0).  Rows keep f; their two source rows s, s + 1 are clamped to the image.  Horizontal
pass in int32, vertical pass with VResizeLinearVec_32s8u's rounding
((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2.
"""
import numpy as np


def _f(ssize, dsize):
    scale = 1.0 / (float(dsize) / float(ssize))
    f = [np.float32((d + 0.5) * scale - 0.5) for d in range(dsize)]
    s = [int(np.floor(v)) for v in f]
    return s, [np.float32(v - np.float32(k)) for v, k in zip(f, s)]


def _coef(f):
    return int(np.rint((np.float32(1) - f) * np.float32(2048))), int(np.rint(f * np.float32(2048)))


def column_table(ssize, dsize):
    """(source column, its coefficient, the next column's) per output column; the next column is min(s + 1, size - 1)."""
    src, c0, c1 = [], [], []
    for s, f in zip(*_f(ssize, dsize)):
        if s < 0:
            s, f = 0, np.float32(0)
        if s >= ssize - 1:
            s, f = ssize - 1, np.float32(0)
        a, b = _coef(f)
        src.append(s); c0.append(a); c1.append(b)
    return np.array(src), np.array(c0), np.array(c1)


def row_table(ssize, dsize):
    """(first source row, second source row, their coefficients) per output row."""
    s, f = _f(ssize, dsize)
    s = np.array(s)
    c = np.array([_coef(v) for v in f])
    return np.clip(s, 0, ssize - 1), np.clip(s + 1, 0, ssize - 1), c[:, 0], c[:, 1]


def resize_linear(img, dst_h, dst_w):
    """uint8 [h,w] or [h,w,C] -> uint8 [dst_h,dst_w(,C)], equal to cv2.resize(img, (dst_w, dst_h))."""
    h, w = img.shape[:2]
    xs, xa0, xa1 = column_table(w, dst_w)
    y0, y1, b0, b1 = row_table(h, dst_h)
    im = img.astype(np.int64).reshape(h, w, -1)
    hr = im[:, xs] * xa0[None, :, None] + im[:, np.minimum(xs + 1, w - 1)] * xa1[None, :, None]
    v = (((b0[:, None, None] * (hr[y0] >> 4)) >> 16) + ((b1[:, None, None] * (hr[y1] >> 4)) >> 16) + 2) >> 2
    return np.clip(v, 0, 255).astype(np.uint8).reshape((dst_h, dst_w) + img.shape[2:])
