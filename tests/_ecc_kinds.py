"""Planes and starting warps W for the ECC certification tests: the kinds of W where an ECC kernel can go wrong (identity,
integer and fractional shifts, the refinement's perturbed H, a horizon through pixel centres, a zero Jacobian
denominator, a mask with a handful of pixels or none, saturating coordinates) and a flat template."""
import cv2
import numpy as np

import _refine_pairs as P

KINDS = ("identity", "shift", "fraction", "perturbed", "horizon", "den0", "handful", "none", "saturate", "flat")


def planes(h, w, seed):
    """-> (template, input) uint8 [h,w]: the refinement's synthetic pair (template = image 2's gray plane, input = image
    1's) where a texture fits, else random bytes."""
    if min(h, w) >= 16:
        img1, img2, _, _ = P.pair(h, w, seed, 3.0)
        return cv2.cvtColor(img2, cv2.COLOR_RGB2GRAY), cv2.cvtColor(img1, cv2.COLOR_RGB2GRAY)
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (h, w), dtype=np.uint8), rng.integers(0, 256, (h, w), dtype=np.uint8)


def warp(kind, h, w, seed=0):
    """W float32 [3,3] of one kind for an h x w plane (W[2,2] = 1 unless stated)."""
    I = np.eye(3)
    if kind in ("identity", "flat"):
        W = I
    elif kind == "shift":
        W = np.array([[1, 0, 3], [0, 1, -2], [0, 0, 1]], np.float64)
    elif kind == "fraction":
        W = np.array([[1, 0, 1.3], [0, 1, -0.7], [0, 0, 1]], np.float64)
    elif kind == "perturbed":                          # the refinement's W_init at the finest level: inv(H_start)
        W = np.linalg.inv(P.pair(h, w, seed, 3.0)[3])
        W /= W[2, 2]
    elif kind == "horizon":                            # W0 = x / 64 - 2: exactly 0 at x = 128, the wl = 0 path
        W = np.array([[1, 0, 0], [0, 1, 0], [1 / 64.0, 0, -2]], np.float64)
    elif kind == "den0":                               # the Jacobian's denominator x W[2,0] + 1 is exactly 0 at x = 64
        W = np.array([[1, 0, 0], [0, 1, 0], [-1 / 64.0, 0, 1]], np.float64)
    elif kind == "handful":                            # only the template's top-left 3 x 2 pixels land in the input
        W = np.array([[1, 0, w - 3], [0, 1, h - 2], [0, 0, 1]], np.float64)
    elif kind == "none":                               # nothing lands in the input: n = 0
        W = np.array([[1, 0, 10 * w], [0, 1, 0], [0, 0, 1]], np.float64)
    elif kind == "saturate":                           # 32 X0 / W0 beyond int32, X >> 5 beyond int16
        W = np.diag([1e6, 1e6, 1.0])
    else:
        raise ValueError(kind)
    return W.astype(np.float32)


def case(kind, h, w, seed=0):
    """-> (template, input, W) for one kind at one size."""
    T, Im = planes(h, w, seed)
    if kind == "flat":
        T = np.full_like(T, 93)
    return T, Im, warp(kind, h, w, seed)
