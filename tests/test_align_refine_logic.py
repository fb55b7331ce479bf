"""Host-side tests of the refinement schedule (align.refine_level_sizes, level_transform, to_level / from_level), its cv2
restatement oracle/ecc_refine.py, the CLI's refinement flags, and the compiled split-pair ECC kernels (no spills; the
one-CTA ECC kernel's SASS unchanged)."""
import hashlib
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _refine_pairs as P  # noqa: E402

cv2 = pytest.importorskip("cv2")


def test_level_sizes():
    from unsuperviseddeephomographyral2018_b200 import align
    S = align.refine_level_sizes
    assert S(240, 320, 3) == [(60, 80), (120, 160), (240, 320)]
    assert S(480, 640, 4) == [(60, 80), (120, 160), (240, 320), (480, 640)]
    assert S(1080, 1920, 4) == [(135, 240), (270, 480), (540, 960), (1080, 1920)]
    assert S(3000, 4000, 5) == [(188, 250), (375, 500), (750, 1000), (1500, 2000), (3000, 4000)]
    assert S(3000, 4000, 1) == [(3000, 4000)]
    # odd sizes halve rounding up, as pyrDown does; a short side below MIN_LEVEL_SIDE ends the pyramid
    assert S(301, 457, 3) == [(76, 115), (151, 229), (301, 457)]
    assert S(33, 1000, 5) == [(17, 500), (33, 1000)]
    assert S(20, 20, 3) == [(20, 20)]
    # max_side scales the finest level (rounded half up), never up
    assert S(3000, 4000, 3, max_side=1000) == [(188, 250), (375, 500), (750, 1000)]
    assert S(1080, 1920, 2, max_side=1001) == [(282, 501), (563, 1001)]
    assert S(240, 320, 2, max_side=1000) == [(120, 160), (240, 320)]
    # levels=None: down to a long side of at most AUTO_COARSEST_SIDE
    assert S(240, 320) == [(240, 320)]
    assert S(480, 640) == [(240, 320), (480, 640)]
    assert S(1080, 1920) == [(135, 240), (270, 480), (540, 960), (1080, 1920)]
    assert S(3000, 4000) == [(188, 250), (375, 500), (750, 1000), (1500, 2000), (3000, 4000)]
    assert S(3000, 4000, max_side=2000) == [(188, 250), (375, 500), (750, 1000), (1500, 2000)]
    for bad in (dict(levels=0), dict(levels=2, max_side=1)):
        with pytest.raises(ValueError):
            S(240, 320, **bad)


@pytest.mark.parametrize("size,size_k", [((480, 640), (240, 320)), ((480, 640), (60, 80)), ((301, 457), (151, 229)),
                                         ((240, 320), (480, 640)), ((3000, 4000), (375, 500))])
def test_level_transform_is_cv2_resize_pixel_map(size, size_k):
    """cv2.resize (INTER_LINEAR) of a linear ramp is the ramp at the mapped coordinates, away from the clamped border."""
    from unsuperviseddeephomographyral2018_b200 import align
    h, w = size
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    a, b, c = 0.37, -0.21, 5.0
    ramp = (a * xs + b * ys + c).astype(np.float32)
    r = cv2.resize(ramp, (size_k[1], size_k[0]))
    Ti = np.linalg.inv(align.level_transform(size, size_k))
    yk, xk = np.mgrid[0:size_k[0], 0:size_k[1]].astype(np.float64)
    X = Ti[0, 0] * xk + Ti[0, 2]
    Y = Ti[1, 1] * yk + Ti[1, 2]
    inner = (X >= 0) & (X <= w - 1) & (Y >= 0) & (Y <= h - 1)
    err = np.abs(r - (a * X + b * Y + c))[inner]
    assert inner.sum() > 0.8 * inner.size and err.max() < 2e-3 * (abs(a) * w + abs(b) * h) / 100, err.max()
    # a pure scale would be off by (s - 1) / 2 px per axis
    assert abs(Ti[0, 2]) > 0 or size == size_k


def test_level_warp_round_trip():
    from unsuperviseddeephomographyral2018_b200 import align
    rng = np.random.default_rng(0)
    for (s1, s2) in (((480, 640), (480, 640)), ((3000, 4000), (3000, 4000)), ((240, 320), (1080, 1920))):
        H = np.stack([P.true_homography(s2[0], s2[1], k) for k in range(4)])
        H[:, :2, :] *= rng.uniform(0.9, 1.1)
        H /= H[:, 2:3, 2:3]
        for sk in align.refine_level_sizes(s2[0], s2[1], 4):
            W = align.to_level(H, s1, s2, sk)
            assert W.dtype == np.float32 and np.all(W[:, 2, 2] == 1)
            back = align.from_level(W, s1, s2, sk)
            for k in range(len(H)):
                # the float32 rounding of W_k moves the corners by at most ~1e-7 of the coordinates
                assert P.corner_error(back[k], H[k], *s1) < 2e-6 * max(s2), (s1, s2, sk)
        # W_k is the level's inverse warp: template pixel -> input pixel
        sk = (s2[0] // 2, s2[1] // 2)
        W = align.to_level(H[:1], s1, s2, sk)[0].astype(np.float64)
        x1 = np.array([[10.0, 20.0], [s1[1] - 5.0, s1[0] / 2.0]])
        x2 = P.apply(H[0], x1)
        T1, T2 = align.level_transform(s1, sk), align.level_transform(s2, sk)
        assert np.abs(P.apply(W, P.apply(T2, x2)) - P.apply(T1, x1)).max() < 1e-3


# Six 480x640 pairs, starting corners off by up to 6 px in the 240x320 frame (12 px here), 3 levels, 50 iterations,
# eps 1e-6: the oracle lands 0.012 to 0.019 px from the true corners (cv2 4.13), so 0.05 px leaves margin for other cv2
# builds.  The residual is the bilinear resampling of warpPerspective's image 2 and its black border, not the schedule.
REFINE_TOL = 0.05


@pytest.mark.parametrize("seed", range(3))
def test_oracle_refines_synthetic_pairs_to_the_truth(seed):
    from oracle import ecc_refine as R
    img1, img2, Ht, H0 = P.pair(480, 640, seed, 6.0)
    assert P.corner_error(H0, Ht, 480, 640) > 5.0
    trace = []
    H, rho, st, lv = R.refine(img1, img2, H0, levels=3, iters=50, eps=1e-6, trace=trace)
    assert (st, lv) == (0, 3) and rho > 0.99
    assert len(trace) == 3 and np.array_equal(trace[-1], H)
    err = P.corner_error(H, Ht, 480, 640)
    print("seed %d: corner error %.4f px" % (seed, err))
    assert err < REFINE_TOL


def test_oracle_failure_keeps_the_previous_H():
    """A pair that raises at a level (here: a flat image 2, NaN correlation) keeps H and reports the status."""
    from oracle import ecc as E, ecc_refine as R
    img1, _, Ht, H0 = P.pair(240, 320, 0, 3.0)
    flat = np.full_like(img1, 77)
    H, rho, st, lv = R.refine(img1, flat, H0, levels=2, iters=10, eps=1e-6)
    assert st in (E.ECC_NAN, E.ECC_NOCONV) and lv == 0 and np.allclose(H, H0 / H0[2, 2], rtol=0, atol=1e-12)


def test_cli_refine_flags():
    import align_images as cli
    a = cli.build_parser().parse_args(["--img1", "a.jpg", "--img2", "b.jpg"])
    assert (a.refine_levels, a.refine_iters, a.refine_eps, a.refine_max_side) == (0, 50, 1e-6, None)
    a = cli.build_parser().parse_args(["--pairs", "p", "--refine_levels", "3", "--refine_iters", "20", "--refine_eps", "1e-5",
                                       "--refine_max_side", "2000"])
    assert (a.refine_levels, a.refine_iters, a.refine_eps, a.refine_max_side) == (3, 20, 1e-5, 2000)


class StubEstimator(object):
    def __init__(self):
        self.refined = []
        self.last_ms = {}

    def estimate(self, I1, I2):
        self.last_ms = dict(prep=1.0, forward=2.0)
        return np.stack([np.eye(3) for _ in I1]), None, None

    def refine(self, I1, I2, H, levels, iters, eps, max_side):
        self.refined.append((len(I1), levels, iters, eps, max_side))
        self.last_ms["refine"] = 4.0
        n = len(I1)
        Hr = np.stack([np.array([[1.0, 0, 0.25 * k], [0, 1.0, -0.5], [0, 0, 1.0]]) for k in range(n)])
        return Hr, np.full(n, 0.98), np.array([0] * (n - 1) + [2], np.int32), np.array([3] * (n - 1) + [1], np.int32)


def _run_cli(tmp_path, extra):
    import align_images as cli
    lst = tmp_path / "pairs.txt"
    lst.write_text("".join("i%d.jpg p%d.jpg\n" % (k, k) for k in range(3)))
    out = tmp_path / ("out%d" % len(extra))
    args = cli.build_parser().parse_args(["--pairs", str(lst), "--out_dir", str(out), "--save_warped", "False"] + extra)
    est = StubEstimator()
    written = cli.run(args, est, lambda paths: [np.zeros((4, 6, 3), np.uint8) for _ in paths], None)
    return est, written, out


def test_cli_refinement_off_by_default_and_on(tmp_path, capsys):
    est, written, out = _run_cli(tmp_path, [])
    assert est.refined == [] and not (out / "refine.txt").exists()
    assert np.array_equal(written, np.tile(np.eye(3, dtype=np.float32).reshape(1, 9), (3, 1)))
    line = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith("===> batch")][0]
    assert "refine" not in line and "(prep 0.333, forward 0.667, warp 0.000)" in line
    est, written, out = _run_cli(tmp_path, ["--refine_levels", "3", "--refine_iters", "7", "--refine_max_side", "900"])
    assert est.refined == [(3, 3, 7, 1e-6, 900)]
    assert np.array_equal(written[:, 2], np.float32([0, 0.25, 0.5]))         # homographies.txt holds the refined H
    assert (out / "refine.txt").read_text().splitlines() == ["i0.jpg p0.jpg 0.98 0 3", "i1.jpg p1.jpg 0.98 0 3",
                                                             "i2.jpg p2.jpg 0.98 2 1"]
    line = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith("===> batch")][0]
    assert "refine 1.333" in line
    est, _, _ = _run_cli(tmp_path, ["--refine_levels", "-1"])
    assert est.refined[0][1] is None


# ---- the compiled kernels -----------------------------------------------------------------------------------------------
def _tool(name):
    p = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), name)
    return p if os.path.exists(p) else shutil.which(name)


NEEDS_TOOLKIT = pytest.mark.skipif(_tool("nvcc") is None or _tool("cuobjdump") is None, reason="the CUDA toolkit is not installed")
ITERATE = "_ZN3udh18ecc_iterate_kernelEPKfS1_idPfPdPiS4_iii"
# sha256 of ecc_iterate_kernel's SASS (instructions and encodings, one per line) as the parent of the split-pair kernels
# compiled it with CUDA 12.9 (V12.9.86) and the library's flags
ITERATE_SASS_SHA256 = {"V12.9.86": "aeebf05e04a06369b5d072b114c4896e3c56765155cc995d41e6367cbe9c4279"}


@pytest.fixture(scope="module")
def ecc_object(tmp_path_factory):
    from unsuperviseddeephomographyral2018_b200 import build_ext
    obj = str(tmp_path_factory.mktemp("ecc") / "ecc.o")
    cmd = [_tool("nvcc")] + build_ext.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build_ext.CSRC, "ecc.cu"), "-o", obj]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, p.stdout
    return obj, p.stdout


def sass_digest(obj, fn):
    sass = subprocess.run([_tool("cuobjdump"), "-sass", "-fun", fn, obj], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                          text=True, timeout=300)
    assert sass.returncode == 0, sass.stdout
    lines = [ln.strip() for ln in sass.stdout.splitlines() if re.match(r"\s+/\*([0-9a-f]{4,}\*/| 0x[0-9a-f]{16} \*/)", ln)]
    assert len(lines) > 1000, sass.stdout[:2000]
    return hashlib.sha256("\n".join(lines).encode()).hexdigest()


@NEEDS_TOOLKIT
def test_split_kernels_do_not_spill(ecc_object):
    _, report = ecc_object
    seen, current = {}, None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current and "ecc_split_" in current:
            seen[current] = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m and current and "ecc_split_" in current:
            print("%s: %s registers" % (current, m.group(1)))
    assert len(seen) == 4, seen                                   # init, stats, jacobian, solve
    assert all(v == (0, 0) for v in seen.values()), seen


@NEEDS_TOOLKIT
def test_one_cta_ecc_kernel_sass_is_unchanged(ecc_object):
    ver = re.search(r"V\d+\.\d+\.\d+", subprocess.run([_tool("nvcc"), "--version"], stdout=subprocess.PIPE, text=True).stdout)
    if not ver or ver.group(0) not in ITERATE_SASS_SHA256:
        pytest.skip("the reference digest was taken with another nvcc (%s)" % (ver.group(0) if ver else "unknown"))
    assert sass_digest(ecc_object[0], ITERATE) == ITERATE_SASS_SHA256[ver.group(0)]
