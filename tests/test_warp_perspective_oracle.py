"""oracle/warp_perspective.py against cv2.warpPerspective on the CPU, byte for byte: cv2 is the only statement of its
rounding we have, so these cases are where the restatement was decided (udh_warp_perspective_u8 is checked against the
restatement on the GPU)."""
import os
import sys

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import warp_perspective as WP  # noqa: E402


def named_matrices(h, w, dh, dw):
    """Identity, translation, mirror, strong perspective, near-singular, singular, a denominator that is zero at output
    column 8 and changes sign inside the output, and maps that send most pixels outside the source."""
    return {
        "identity": np.eye(3),
        "translation": np.array([[1, 0, 3.37], [0, 1, -2.25], [0, 0, 1.0]]),
        "mirror": np.array([[-1, 0, w - 1], [0, 1, 0], [0, 0, 1.0]]),
        "perspective": np.array([[0.9, 0.2, 5], [-0.1, 1.1, 3], [0.004, 0.003, 1.0]]),
        "near_singular": np.array([[1, 2, 3], [2, 4 + 1e-9, 6], [0.001, 0.002, 1.0]]),
        "singular": np.array([[1, 2, 0], [2, 4, 0], [0, 0, 1.0]]),
        "zero_denominator": np.array([[1, 0, 0], [0, 1, 0], [0.125, 0, 1.0]]),
        "denominator_crosses_zero": np.array([[1, 0.1, 0], [0.05, 1, 0], [2.0 / max(dw, 2), 0.001, 1.0]]),  # inverse's: 1 - 2x/dw
        "mostly_outside": np.array([[1, 0, 0.8 * w], [0, 1, -0.7 * h], [0, 0, 1.0]]),
        "shrink_far": np.array([[0.05, 0, 4 * w], [0, 0.05, 0], [0, 0, 1.0]]),
    }


def _diff(a, b):
    d = np.argwhere((a != b).reshape(a.shape[0], a.shape[1], -1).any(-1))
    return "%d pixels differ, first at %s: cv2 %s oracle %s" % (len(d), d[0].tolist(), a[tuple(d[0])], b[tuple(d[0])])


SIZES = [((1, 1), (1, 1)), ((1, 1), (5, 7)), ((2, 3), (3, 2)), ((17, 23), (9, 11)), ((17, 23), (40, 60)),
         ((60, 80), (60, 80)), ((240, 320), (142, 190)), ((142, 190), (480, 640)), ((480, 640), (240, 320)), ((480, 640), (480, 640))]


@pytest.mark.parametrize("channels", [1, 3], ids=["gray", "bgr"])
@pytest.mark.parametrize("src_hw,dst_hw", SIZES, ids=["%dx%d_to_%dx%d" % (a + b) for a, b in SIZES])
def test_named_matrices(channels, src_hw, dst_hw):
    (h, w), (dh, dw) = src_hw, dst_hw
    rng = np.random.default_rng(h * 1000 + w + dh + channels)
    src = rng.integers(0, 256, (h, w, channels) if channels == 3 else (h, w), np.uint8)
    for name, M in named_matrices(h, w, dh, dw).items():
        a = cv2.warpPerspective(src, M, (dw, dh))
        b = WP.warp_perspective(src, M, (dw, dh))
        assert a.shape == b.shape and np.array_equal(a, b), "%s: %s" % (name, _diff(a, b))


def test_seeded_random_matrices():
    rng = np.random.default_rng(2026)
    for k in range(200):
        h, w = int(rng.integers(1, 160)), int(rng.integers(1, 160))
        dh, dw = int(rng.integers(1, 200)), int(rng.integers(1, 200))
        src = rng.integers(0, 256, (h, w, 3) if k % 2 else (h, w), np.uint8)
        M = np.eye(3) + rng.normal(0, 0.1, (3, 3)) * [[1, 1, 20], [1, 1, 20], [0.003, 0.003, 0.1]]
        a = cv2.warpPerspective(src, M, (dw, dh))
        b = WP.warp_perspective(src, M, (dw, dh))
        assert np.array_equal(a, b), "case %d: %s" % (k, _diff(a, b))


def test_zero_denominator_lands_on_the_first_source_pixel():
    """Where W = 0 the source position is (0, 0) in cv2, not the border: the restatement keeps that."""
    src = np.full((20, 30, 3), 7, np.uint8)
    src[0, 0] = (200, 100, 50)
    out = WP.warp_perspective(src, np.array([[1, 0, 0], [0, 1, 0], [0.125, 0, 1.0]]), (30, 20))
    assert (out[:, 8] == (200, 100, 50)).all()
    assert np.array_equal(out, cv2.warpPerspective(src, np.array([[1, 0, 0], [0, 1, 0], [0.125, 0, 1.0]]), (30, 20)))
