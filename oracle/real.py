"""NumPy restatement of the real-data direct-method metric (code/homography_conventional_real.py:213-246 with
code/utils/direct_homography.py:42-57, return_h_inv=False), the arithmetic udh_ecc_corr_h4p runs (test infrastructure).

Per sample, gt holds the 16 clicked numbers (fp32, 480x640 frame): corr1 = gt[0:8] / 2, corr2 = gt[8:16] / 2.
  found:     pred = perspectiveTransform(corr1, W) - corr1 in fp32 (cv2 transforms in double with the matrix widened to
             double, |w| <= FLT_EPSILON gives 0), clamped to +-80; h = sqrt(mean(square(pred + corr1 - corr2))) in fp32
             (NumPy's pairwise sum of the 8 squares); fail 2 and h = the identity error when that is smaller.
  not found: pred = float64 zeros, so h = the identity error in float64, fail 1.
"""
import numpy as np

FLT_EPSILON = float(np.finfo(np.float32).eps)


def _rmse32(d):
    s = np.square(d.reshape(-1).astype(np.float32))
    t = ((s[0] + s[1]) + (s[2] + s[3])) + ((s[4] + s[5]) + (s[6] + s[7]))          # numpy pairwise_sum, n = 8
    return np.sqrt(np.float32(t / np.float32(8)))


def perspective_transform_f32(pts, W):
    m = np.asarray(W, np.float32).astype(np.float64).reshape(9)
    out = np.zeros_like(pts, dtype=np.float32)
    for k, (x, y) in enumerate(np.asarray(pts, np.float32).astype(np.float64)):
        w = x * m[6] + y * m[7] + m[8]
        if abs(w) > FLT_EPSILON:
            w = 1.0 / w
            out[k] = [np.float32((x * m[0] + y * m[1] + m[2]) * w), np.float32((x * m[3] + y * m[4] + m[5]) * w)]
    return out


def corr_h4p(W, status, gt):
    """W [B,3,3] fp32, status [B] (nonzero: ECC raised), gt [B,16] fp32 -> (pred [B,8] fp32, h [B] float64, fail [B] int32)."""
    W, gt = np.asarray(W, np.float32).reshape(-1, 3, 3), np.asarray(gt, np.float32)
    B = len(W)
    pred, h, fail = np.zeros((B, 8), np.float32), np.zeros(B, np.float64), np.zeros(B, np.int32)
    for b in range(B):
        c1 = (gt[b, 0:8] / np.float32(2)).reshape(4, 2)
        c2 = (gt[b, 8:16] / np.float32(2)).reshape(4, 2)
        if status[b] != 0:
            d = c1.astype(np.float64) - c2.astype(np.float64)
            h[b], fail[b] = np.sqrt(np.mean(np.square(d))), 1
            continue
        p = perspective_transform_f32(c1, W[b]) - c1
        p[p >= 80] = 80
        p[p <= -80] = -80
        pred[b] = p.reshape(8)
        hv, hi = _rmse32((p + c1) - c2), _rmse32(c1 - c2)
        if hi < hv:
            hv, fail[b] = hi, 2
        h[b] = float(hv)
    return pred, h, fail
