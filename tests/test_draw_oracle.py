"""oracle/draw.py against cv2 on the CPU: every drawing primitive of the report image, and the report's composition, byte
for byte.  cv2 is the only statement of these rules we have, so each test here is where one of them was decided."""
import os
import sys

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import draw as D  # noqa: E402
from unsuperviseddeephomographyral2018_b200 import report  # noqa: E402


def background(rng, h, w, noise):
    return rng.integers(0, 256, (h, w, 3), np.uint8) if noise else np.full((h, w, 3), 131, np.uint8)


def _diff(a, b):
    d = np.argwhere((a != b).any(-1))
    return "%d pixels differ, first at %s: cv2 %s oracle %s" % (len(d), d[0].tolist(), a[tuple(d[0])], b[tuple(d[0])])


# 2 backgrounds x 2 sizes x 150 sets x 15 primitives = 9000 primitives
@pytest.mark.parametrize("noise", [True, False], ids=["noise", "constant"])
@pytest.mark.parametrize("hw", [(17, 23), (40, 60)], ids=["17x23", "40x60"])
def test_primitives(noise, hw):
    h, w = hw
    rng = np.random.default_rng(100 + noise + 2 * w)
    cases = D.vertex_cases(rng, 150, h, w)
    for k, v in enumerate(cases):
        img = background(rng, h, 2 * w, noise)
        col = tuple(int(c) for c in rng.integers(0, 256, 3))
        for s in (0, 4, 8):                                        # [test_thick_polyline] [test_fill_convex_poly]
            a = img.copy(); cv2.polylines(a, [v[s:s + 4]], True, col, 3)
            b = img.copy(); D.polylines_closed(b, v[s:s + 4], col)
            assert np.array_equal(a, b), "case %d polyline %s: %s" % (k, v[s:s + 4].tolist(), _diff(a, b))
        for i in range(4):                                         # [test_line_aa] [test_circle_aa]
            p, q = tuple(int(c) for c in v[12 + i]), tuple(int(c) for c in v[16 + i])
            a = img.copy(); cv2.line(a, p, q, col, 1, cv2.LINE_AA)
            b = img.copy(); D.line(b, p, q, col)
            assert np.array_equal(a, b), "case %d line %s %s: %s" % (k, p, q, _diff(a, b))
            for c in (p, q):
                a = img.copy(); cv2.circle(a, c, 7, col, 1, cv2.LINE_AA)
                b = img.copy(); D.circle(b, c, 7, col)
                assert np.array_equal(a, b), "case %d circle %s: %s" % (k, c, _diff(a, b))


def test_extreme_vertices():
    """Every pair of the int32 extremes and a point on the image, in both directions, as thick edges and AA lines."""
    h, w = 17, 46
    rng = np.random.default_rng(7)
    pts = [(x, y) for x in D.EXTREMES + [5] for y in D.EXTREMES + [9]]
    img = background(rng, h, w, True)
    for p in pts:
        for q in [(5, 9), (40, 2), (-4, 20)]:
            a = img.copy(); cv2.polylines(a, [np.int32([p, q, (3, 3)])], True, (9, 99, 199), 3)
            b = img.copy(); D.polylines_closed(b, np.int32([p, q, (3, 3)]), (9, 99, 199))
            assert np.array_equal(a, b), "polyline %s %s: %s" % (p, q, _diff(a, b))
            a = img.copy(); cv2.line(a, p, q, (9, 99, 199), 1, cv2.LINE_AA)
            b = img.copy(); D.line(b, p, q, (9, 99, 199))
            assert np.array_equal(a, b), "line %s %s: %s" % (p, q, _diff(a, b))
        a = img.copy(); cv2.circle(a, p, 7, (9, 99, 199), 1, cv2.LINE_AA)
        b = img.copy(); D.circle(b, p, 7, (9, 99, 199))
        assert np.array_equal(a, b), "circle %s: %s" % (p, _diff(a, b))


def test_line_aa_visits_each_pixel_once():
    """One LineAA segment blends each pixel at most once (each step has its own major coordinate), so its pixels may be
    blended in any order; cv2 agreeing with the oracle on noise backgrounds (test_primitives) pins the blend itself."""
    rng = np.random.default_rng(3)
    for v in D.vertex_cases(rng, 300, 40, 60):
        for i in range(4):
            px = D.line_aa_pixels(120, 40, *(int(c) << D.XY_SHIFT for c in (*v[12 + i], *v[16 + i])))
            assert len(px) == len({(x, y) for x, y, _ in px})
        for (x0, y0), (x1, y1) in zip(D.circle_poly(int(v[12, 0]), int(v[12, 1]), 7)[:-1], D.circle_poly(int(v[12, 0]), int(v[12, 1]), 7)[1:]):
            px = D.line_aa_pixels(120, 40, x0, y0, x1, y1)
            assert len(px) == len({(x, y) for x, y, _ in px})


def test_circle_polygon():
    """ellipse2Poly for r = 7: 13 vertices (0..360 step 30, the first repeated last), integer centre."""
    v = D.circle_poly(10, 20, 7)
    assert len(v) == 13 and v[0] == v[-1] == (17 << 16, 20 << 16)
    assert v[3] == (10 << 16, 27 << 16)


@pytest.mark.parametrize("hw", [(240, 320), (17, 23)], ids=["240x320", "17x23"])
@pytest.mark.parametrize("noise", [True, False], ids=["noise", "constant"])
def test_composition(hw, noise):
    """The report from float points: report.report_vertices + the oracle's drawing == the cv2 call sequence with the
    reference's own conversions, and so are the JPEG bytes."""
    h, w = hw
    rng = np.random.default_rng(11 + h)
    for k in range(12):
        img1, img2 = background(rng, h, w, noise), background(rng, h, w, noise)
        corr1 = (rng.uniform(-0.2, 1.2, (4, 2)) * [w, h]).astype(np.float32)
        corr2 = (corr1 + rng.normal(0, 0.1 * w, (4, 2))).astype(np.float32)
        pred = (corr2 + rng.normal(0, 0.05 * w, (4, 2))).astype(np.float32)
        if k % 4 == 1:
            corr2 = np.round(corr2.astype(np.float64)) + 0.5        # exact halves: np.round is half-to-even
            pred[rng.integers(0, 4)] = np.nan                        # np.int32(nan) = INT_MIN
        if k % 4 == 2:
            pred = pred * 1e4                                        # far outside the canvas
        with np.errstate(invalid="ignore"):
            ref = D.cv2_compose(img1, img2, corr1, corr2, pred)
        out = D.draw_report(img1, img2, report.report_vertices(corr1, corr2, pred, w))
        assert np.array_equal(ref, out), "case %d: %s" % (k, _diff(ref, out))
        assert cv2.imencode(".jpg", ref)[1].tobytes() == cv2.imencode(".jpg", out)[1].tobytes()


def test_vertex_sets_against_cv2():
    """The composition from the seeded vertex sets the GPU test also draws."""
    rng = np.random.default_rng(5)
    for h, w in ((17, 23), (48, 64)):
        for v in D.vertex_cases(rng, 60, h, w):
            img1, img2 = background(rng, h, w, True), background(rng, h, w, True)
            ref = D.cv2_draw_report(img1, img2, v)
            out = D.draw_report(img1, img2, v)
            assert np.array_equal(ref, out), _diff(ref, out)
