"""CPU tests of the direct-method baseline's NumPy restatement (oracle/ecc.py) against OpenCV, and of the new C entry
points' failure mode without a GPU.  The OpenCV comparisons skip only when cv2 is not installed."""
import os
import zlib

import numpy as np
import pytest
import torch

from oracle import ecc as E
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ecc_golden.npz")
AUG0 = [1, 1.1, 1.3, 0.9, 1.05, 1.15, 0.85, 0.7, 1.1, 0.95, 1.0]


def _cv2():
    return pytest.importorskip("cv2")


def _pairs():
    """12 rho = 45 pairs of oracle.make_batch(seed=3), sample 0 augmented."""
    b = O.make_batch(3, 12)
    aug = np.zeros((12, 11), np.float32); aug[0] = AUG0
    return b, aug


def _smooth_pair():
    """A smooth texture under a small warp: ECC converges on it."""
    ys, xs = np.mgrid[0:240, 0:320].astype(np.float64)
    img = 128 + 60 * np.sin(xs / 17.0) * np.cos(ys / 23.0) + 30 * np.sin((xs + ys) / 41.0)
    t = np.clip(img, 0, 255).astype(np.uint8)
    Wt = np.array([[1.0, 0.004, 1.6], [-0.003, 1.0, -1.2], [0.0, 0.0, 1.0]], np.float32)
    return t, np.clip(E.warp_linear(img.astype(np.float32), np.linalg.inv(Wt)), 0, 255).astype(np.uint8)


def _cv_ecc(cv2, t, im, k):
    try:
        rho, W = cv2.findTransformECC(t, im, np.eye(3, dtype=np.float32), cv2.MOTION_HOMOGRAPHY,
                                      (cv2.TERM_CRITERIA_EPS | cv2.TERM_CRITERIA_COUNT, k, 1e-10), None, 5)
        return W, rho, E.ECC_OK
    except cv2.error as e:
        return None, None, E.ECC_NAN if "NaN" in str(e) else E.ECC_NOCONV


def test_gray_planes_match_the_reference_round_trip():
    cv2 = _cv2()
    b, aug = _pairs()
    g1, g2 = E.prep(b["I_u8"][:2], b["I_prime_u8"][:2], aug[:2])
    for s, img, g in ((0, b["I_u8"], g1), (1, b["I_u8"], g1), (0, b["I_prime_u8"], g2), (1, b["I_prime_u8"], g2)):
        five = (aug[s, 1:6] if img is b["I_u8"] else aug[s, 6:11]) if aug[s, 0] else None
        n = E.augment_normalise(img[s], five)
        ref = cv2.cvtColor((n * np.array(E.STD).reshape(1, 1, 3) + np.array(E.MEAN).reshape(1, 1, 3)).astype(np.uint8), cv2.COLOR_RGB2GRAY)
        assert np.array_equal(ref, g[s])
    # the round trip is not the identity: about half the bytes of a plain image come back one lower
    plain = E.denorm_u8(E.augment_normalise(b["I_u8"][1]))
    frac = (plain == b["I_u8"][1]).mean()
    assert 0.2 < frac < 0.8 and ((plain.astype(int) - b["I_u8"][1]) >= -1).all()


def test_blur_gradients_and_warp_match_opencv():
    cv2 = _cv2()
    b, aug = _pairs()
    g = E.prep(b["I_u8"][:1], b["I_prime_u8"][:1], aug[:1])[1][0]
    bl = cv2.GaussianBlur(g.astype(np.float32), (5, 5), 0, 0)
    assert np.array_equal(bl, E.blur(g))
    gx, gy = E.gradients(bl)
    assert np.array_equal(gx, cv2.filter2D(bl, -1, np.array([[-0.5, 0, 0.5]], np.float32)))
    assert np.array_equal(gy, cv2.filter2D(bl, -1, np.array([[-0.5], [0], [0.5]], np.float32)))
    for Wt in (np.array([[1.01, 0.02, 3.3], [-0.015, 0.99, -2.7], [1e-5, -2e-5, 1.0]], np.float32),
               np.array([[0.8, 0.1, 40.0], [0.05, 1.2, -30.0], [3e-4, -2e-4, 1.0]], np.float32)):
        ref = cv2.warpPerspective(bl, Wt, (320, 240), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP)
        assert np.abs(ref - E.warp_linear(bl, Wt)).max() <= 1e-5 * np.abs(ref).max()


def _w_close(Wa, Wb, H=240, Wd=320):
    """Largest distance (px) between where Wa and Wb send the template's four corners."""
    c = np.array([[0, 0, 1], [Wd - 1, 0, 1], [Wd - 1, H - 1, 1], [0, H - 1, 1]], np.float64).T
    pa = Wa.astype(np.float64) @ c; pb = Wb.astype(np.float64) @ c
    return float(np.abs(pa[:2] / pa[2] - pb[:2] / pb[2]).max())


# Pairs whose outcome is decided by a quantity within 1e-4 relative of its threshold: none in this set (the smallest
# |lambda_d| / |correlation| on a deciding iteration is 0.74).
AMBIGUOUS = ()


@pytest.mark.parametrize("k", [1, 2, 8])
def test_iterations_match_opencv(k):
    """W after k iterations (cv2 run with maxCount = k).  Status and iteration count match on every pair; W agrees to
    0.1 px at the corners after one iteration (the worst pair, rho = 0.003, is at 0.05 px: cv2 inverts a float32 Hessian) and, on the converging pair, after k.  The rho = 45 pairs that do not
    raise diverge (rho ~ 0.05): their later iterates amplify float32 rounding and are compared on status only."""
    cv2 = _cv2()
    b, aug = _pairs()
    g1, g2 = E.prep(b["I_u8"], b["I_prime_u8"], aug)
    t, im = _smooth_pair()
    cases = [(g1[s], g2[s], False) for s in range(12)] + [(t, im, True)]
    seen = set()
    for j, (a, c, converging) in enumerate(cases):
        W, rho, st = _cv_ecc(cv2, a, c, k)
        tr = []
        o = E.ecc(a, c, max_iters=k, solve="fp32", trace=tr)
        seen.add(st)
        if j in AMBIGUOUS:
            continue
        # the deciding quantity of each iteration: rho (NaN or not: exact) and lambda_d against 0
        assert all(np.isnan(x["rho"]) or abs(x["lambda_d"]) > 1e-4 * abs(x["corr"]) for x in tr), j
        assert o["status"] == st, (j, o["status"], st)
        if st == E.ECC_OK:
            assert o["iters"] == k
            if k == 1 or converging:
                assert _w_close(W, o["W"]) < 0.1, (j, _w_close(W, o["W"]))
            assert abs(o["rho"] - rho) < 1e-3 * max(1.0, abs(rho)) or not (k == 1 or converging)
        if converging:
            assert st == E.ECC_OK and rho > 0.9
    assert E.ECC_OK in seen and E.ECC_NOCONV in seen


def test_golden_file_matches_the_oracle():
    """ecc_golden.npz: cv2's outcome on regenerated inputs (tests/golden/make_ecc_golden.py)."""
    z = np.load(GOLDEN)
    b, aug = _pairs()
    g1, g2 = E.prep(b["I_u8"], b["I_prime_u8"], aug)
    assert zlib.crc32(g1.tobytes()) == int(z["crc_gray_I"]) and zlib.crc32(g2.tobytes()) == int(z["crc_gray_I_prime"])
    for s in range(len(z["status"])):
        o = E.ecc(g1[s], g2[s], max_iters=int(z["max_iters"]), solve="fp32")
        assert o["status"] == int(z["status"][s])
        if o["status"] == E.ECC_OK:
            assert o["iters"] == int(z["max_iters"])


def test_h4p_post_processing_rules():
    pts = np.array([100, 50, 228, 50, 228, 178, 100, 178], np.float32)
    gt = np.array([3, -2, 1, 4, -5, 2, 0, 1], np.float32)
    W = np.array([[1, 0, -3.0], [0, 1, 2.0], [0, 0, 1]], np.float32)        # inv(W) shifts by (+3, -2)
    pred, hl, fail = E.h4p(W, E.ECC_OK, pts, gt)
    assert np.allclose(pred, [3, -2] * 4, atol=1e-4) and fail == 2 and hl == pytest.approx(np.sqrt(np.mean(gt.astype(float) ** 2)))
    pred, hl, fail = E.h4p(W, E.ECC_NOCONV, pts, gt)
    assert not pred.any() and fail == 1
    Wbig = np.array([[1, 0, -50.0], [0, 1, 0], [0, 0, 1]], np.float32)
    pred, _, _ = E.h4p(Wbig, E.ECC_OK, pts, gt)
    assert (pred[0::2] == 90).all()
    pred, hl, fail = E.h4p(np.eye(3, dtype=np.float32), E.ECC_OK, pts, gt)
    assert fail == 0 and hl == pytest.approx(np.sqrt(np.mean(gt.astype(float) ** 2)))   # identity == identity: not a failure


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_ecc_entry_points_fail_cleanly_without_a_gpu():
    from unsuperviseddeephomographyral2018_b200 import _lib, direct_homography, ops
    assert _lib.lib.udh_ecc_workspace_bytes(2, 240, 320) == 2 * 2 * 240 * 320 * 4
    with pytest.raises(_lib.UdhError):
        ops.ecc_prep_u8(torch.zeros(1, 8, 8, 3, dtype=torch.uint8), torch.zeros(1, 8, 8, 3, dtype=torch.uint8))
    with pytest.raises(_lib.UdhError):
        ops.find_homography_ecc(torch.zeros(1, 8, 8, dtype=torch.uint8), torch.zeros(1, 8, 8, dtype=torch.uint8))
    with pytest.raises(_lib.UdhError):
        direct_homography.find_homography(torch.zeros(1, 8, 8, dtype=torch.uint8), torch.zeros(1, 8, 8, dtype=torch.uint8),
                                          torch.zeros(1, 8))
    assert _lib.lib.udh_ecc_h4p(None, None, None, None, 45.0, None, None, None, 1, None) == _lib.EINVAL
