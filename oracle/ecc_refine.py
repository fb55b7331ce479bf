"""cv2 restatement of align.HomographyEstimator.refine: coarse-to-fine cv2.findTransformECC on the images' own pixels.

Level sizes and the float64 coordinate conjugations are align's (refine_level_sizes, to_level, from_level), so the two
agree exactly at level boundaries; the planes and the iterations are cv2's: cvtColor(cv2.resize(img, (w_k, h_k)),
RGB2GRAY) and findTransformECC(template = image 2's plane, input = image 1's, W_k, MOTION_HOMOGRAPHY, (COUNT | EPS,
iters, eps), None, 5).  A cv2 exception ends the pair with the status it stands for (ecc.ECC_NAN for "NaN encountered",
ecc.ECC_NOCONV for "stopped before its convergence") and the H it had before that level.  Test-only: no GPU.
"""
import cv2
import numpy as np

from oracle import ecc as E
from unsuperviseddeephomographyral2018_b200 import align


def level_plane(img_rgb, size_k):
    r = img_rgb if img_rgb.shape[:2] == tuple(size_k) else cv2.resize(img_rgb, (size_k[1], size_k[0]))
    return cv2.cvtColor(r, cv2.COLOR_RGB2GRAY)


def ecc_status(err):
    msg = str(err)
    if "NaN encountered" in msg:
        return E.ECC_NAN
    if "stopped before its convergence" in msg:
        return E.ECC_NOCONV
    raise err


def refine(img1, img2, H, levels=align.REFINE_LEVELS, iters=align.REFINE_ITERS, eps=align.REFINE_EPS, max_side=None, trace=None):
    """One pair: uint8 RGB img1 [h1,w1,3], img2 [h2,w2,3], H [3,3] (image 1 -> image 2) -> (H float64 [3,3], rho, status,
    level_reached).  `trace` (a list) receives H after every level that succeeded."""
    s1, s2 = img1.shape[:2], img2.shape[:2]
    H = np.asarray(H, np.float64).reshape(1, 3, 3)
    H = H / H[0, 2, 2]
    rho, status, reached = float("nan"), E.ECC_OK, 0
    crit = (cv2.TERM_CRITERIA_COUNT | cv2.TERM_CRITERIA_EPS, iters, eps)
    for lv, sk in enumerate(align.refine_level_sizes(s2[0], s2[1], levels, max_side)):
        W = align.to_level(H, s1, s2, sk)[0]
        try:
            rho, W = cv2.findTransformECC(level_plane(img2, sk), level_plane(img1, sk), W, cv2.MOTION_HOMOGRAPHY, crit, None, 5)
        except cv2.error as err:
            status, rho = ecc_status(err), float("nan")
            break
        H = align.from_level(W[None], s1, s2, sk)
        reached = lv + 1
        if trace is not None:
            trace.append(H[0].copy())
    return H[0], rho, status, reached
