"""Host-side tests of the mosaic's multi-band blend: the NumPy restatement (oracle/multiband.py) against cv2's pyramids and
cv2.detail_MultiBandBlender byte for byte, the ROI rule against the full-canvas validity map, mosaic_images.py's --blend
and --bands, and the compiled kernels (no spills; the warp and feathered-blend kernels' SASS unchanged)."""
import hashlib
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _mosaic_sweep as SW  # noqa: E402

cv2 = pytest.importorskip("cv2")
from oracle import mosaic as OM  # noqa: E402
from oracle import multiband as MB  # noqa: E402


# ---- pyramids ----------------------------------------------------------------------------------------------------------------
SIDES = list(range(1, 10)) + [16, 31, 64, 101]


@pytest.mark.parametrize("dtype", [np.uint8, np.int16])
@pytest.mark.parametrize("C", [1, 3])
def test_pyramids_equal_cv2(dtype, C):
    rng = np.random.default_rng(C)
    for H in SIDES:
        for W in SIDES:
            shape = (H, W) if C == 1 else (H, W, 3)
            a = rng.integers(0, 256, shape) if dtype == np.uint8 else rng.integers(-32768, 32768, shape)
            a = a.astype(dtype)
            assert np.array_equal(MB.pyr_down(a), cv2.pyrDown(a)), ("pyrDown", H, W)
            assert np.array_equal(MB.pyr_up(a), cv2.pyrUp(a)), ("pyrUp", H, W)


def test_pyr_up_right_edge_is_not_reflect_101():
    s = np.array([[20, 60, 100]], np.uint8).repeat(2, 0)
    assert list(cv2.pyrUp(s)[0]) == list(MB.pyr_up(s)[0]) == [30, 40, 60, 80, 95, 100]    # 95 = (60 + 7 100) / 8


# ---- the restatement against cv2's blender -------------------------------------------------------------------------------
def _random_feeds(rng, Hc, Wc, rects, fill=0.8):
    imgs, masks, tls = [], [], []
    for x, y, w, h in rects:
        assert 0 <= x and x + w <= Wc and 0 <= y and y + h <= Hc
        imgs.append(rng.integers(0, 256, (h, w, 3), np.uint8))
        masks.append(np.where(rng.random((h, w)) < fill, 255, 0).astype(np.uint8))
        tls.append((x, y))
    return imgs, masks, tls


def _check(Hc, Wc, bands, rects, seed=0, fill=0.8):
    imgs, masks, tls = _random_feeds(np.random.default_rng(seed), Hc, Wc, rects, fill)
    r = MB.restate(imgs, masks, tls, Hc, Wc, bands)
    out, mask, dst = MB.cv2_blend(imgs, masks, tls, Hc, Wc, bands)
    assert np.array_equal(r["dst"], dst) and np.array_equal(r["mask"], mask) and np.array_equal(r["mosaic"], out)
    return r, dst


EDGES = [(0, 0, 40, 30), (45, 0, 40, 30), (91, 0, 40, 30), (0, 33, 40, 30), (91, 33, 40, 30), (0, 67, 40, 30), (45, 67, 40, 30),
         (91, 67, 40, 30), (50, 20, 5, 3), (3, 90, 2, 7)]


@pytest.mark.parametrize("bands", [0, 1, 2, 5, 8])
def test_restatement_equals_cv2_at_every_edge_and_corner(bands):
    """tl at every canvas edge and corner, ROIs far smaller than the gap, a 97 x 131 canvas (not a multiple of 2^B)."""
    r, dst = _check(97, 131, bands, EDGES, seed=bands)
    assert r["bands"] == bands
    assert dst.min() < 0 or dst.max() > 255 or bands == 0          # the saturation to uint8 matters


@pytest.mark.parametrize("Hc,Wc,bands,want", [(20, 30, 8, 5), (16, 16, 10, 4), (17, 16, 10, 5), (1, 1, 3, 0), (3, 200, 10, 8)])
def test_restatement_clips_the_bands_to_the_canvas(Hc, Wc, bands, want):
    r, _ = _check(Hc, Wc, bands, [(0, 0, min(Wc, 7), min(Hc, 5)), (Wc - min(Wc, 4), Hc - min(Hc, 3), min(Wc, 4), min(Hc, 3))])
    assert r["bands"] == want


def test_restatement_equals_cv2_with_full_masks_and_odd_sides():
    _check(211, 157, 5, [(0, 0, 157, 211), (30, 40, 100, 120), (100, 150, 57, 61)], seed=4, fill=1.0)


def test_single_frame_normalises_by_w_plus_1():
    """A lone flat frame does not come back: each level is scaled by 256 / 257 and truncated, so 255 -> 254 and 200 -> 199
    at 0 bands, and lower still where more levels lose their fraction."""
    for bands in (0, 5):
        for v in (255, 200):
            img = np.full((40, 50, 3), v, np.uint8)
            r = MB.restate([img], [np.full((40, 50), 255, np.uint8)], [(0, 0)], 40, 50, bands)
            out, _, _ = MB.cv2_blend([img], [np.full((40, 50), 255, np.uint8)], [(0, 0)], 40, 50, bands)
            assert np.array_equal(r["mosaic"], out) and out.max() <= v - 1
            assert np.all(out == v - 1) or bands > 0


def test_restatement_equals_cv2_where_the_sums_wrap():
    """131 frames over one spot: the int16 weight sum passes 32767 (131 x 256) and wraps, in acc too."""
    rects = [(2 + k % 5, 3 + k % 3, 30, 24) for k in range(131)]
    r, _ = _check(33, 41, 3, rects, seed=9, fill=1.0)
    assert (r["wacc"][0] < 0).any() and (r["mask"] == 0).any()


def test_feed_order_and_dtype_do_not_matter():
    imgs, masks, tls = _random_feeds(np.random.default_rng(5), 97, 131, EDGES)
    a = MB.cv2_blend(imgs, masks, tls, 97, 131, 5)[2]
    p = list(range(len(imgs)))[::-1]
    b = MB.cv2_blend([imgs[k] for k in p], [masks[k] for k in p], [tls[k] for k in p], 97, 131, 5)[2]
    c = MB.cv2_blend([i.astype(np.int16) for i in imgs], masks, tls, 97, 131, 5)[2]
    assert np.array_equal(a, b) and np.array_equal(a, c)


# ---- the ROI rule --------------------------------------------------------------------------------------------------------------
def _roi_holds_every_valid_pixel(frames, M, Hc, Wc):
    from unsuperviseddeephomographyral2018_b200 import mosaic
    rois, Mr = mosaic.multiband_rois(M, [f.shape[:2] for f in frames], Hc, Wc)
    for k, f in enumerate(frames):
        h, w = f.shape[:2]
        valid, _ = OM.validity_weight(M[k], h, w, Hc, Wc, 0)
        x0, y0, x1, y1 = rois[k]
        inside = np.zeros_like(valid)
        inside[y0:y1, x0:x1] = True
        assert not (valid & ~inside).any(), k
        assert np.allclose(Mr[k], np.array([[1.0, 0, -x0], [0, 1.0, -y0], [0, 0, 1.0]]) @ M[k], rtol=0, atol=0)


@pytest.mark.parametrize("name", ["one", "two", "seven"])
def test_roi_holds_every_valid_pixel_of_the_named_cases(name):
    import test_gpu_mosaic as GM
    frames, M, (Hc, Wc) = GM._case(name, 3, np.random.default_rng(0))
    _roi_holds_every_valid_pixel(frames, M, Hc, Wc)


@pytest.mark.parametrize("n,h,w,seed", [(6, 240, 320, 2), (4, 1080, 1920, 4)])
def test_roi_holds_every_valid_pixel_of_a_sweep(n, h, w, seed):
    from unsuperviseddeephomographyral2018_b200 import mosaic
    A, _ = SW.sweep_cameras(n, h, w, 0.6, seed)
    G, ref = mosaic.chain_to_reference(SW.true_pairs(A))
    M, (Hc, Wc), kept = mosaic.canvas([(h, w)] * n, G, ref)
    _roi_holds_every_valid_pixel([np.zeros((h, w, 3), np.uint8)] * n, M, Hc, Wc)


def test_roi_rejects_frames_behind_the_camera():
    from unsuperviseddeephomographyral2018_b200 import mosaic
    for M in (np.array([[1.0, 0, 0], [0, 1.0, 0], [-0.2, 0, 1.0]]), np.full((3, 3), np.inf)):
        with pytest.raises(ValueError):
            mosaic.multiband_rois(M[None], [(8, 8)], 8, 8)


# ---- the CLI ---------------------------------------------------------------------------------------------------------------
def test_cli_blend_flags():
    import mosaic_images as cli
    a = cli.build_parser().parse_args(["--frames", "raw"])
    assert (a.blend, a.bands, a.feather) == ("feather", 5, 64)
    a = cli.build_parser().parse_args(["--frames", "raw", "--blend", "multiband", "--bands", "8"])
    assert (a.blend, a.bands) == ("multiband", 8)
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args(["--frames", "raw", "--blend", "laplace"])
    for bands in (-1, 11):
        with pytest.raises(SystemExit):
            cli.run(cli.build_parser().parse_args(["--frames", "raw", "--blend", "multiband", "--bands", str(bands)]), None, None, None)


@pytest.mark.parametrize("blend", ["feather", "multiband"])
def test_cli_mosaic_txt(tmp_path, monkeypatch, blend):
    """mosaic.txt as run() writes it from build_mosaic's result: the feathered blend's is the parent's format, the
    multi-band one's first line names the blend and its bands."""
    import torch
    import mosaic_images as cli
    from unsuperviseddeephomographyral2018_b200 import mosaic
    raw = tmp_path / "raw"
    raw.mkdir()
    for k in range(3):
        (raw / ("F_%d.JPG" % k)).write_bytes(b"")
    seen = {}

    def fake_build(est, imgs, ref, refine, feather, float32_M=False, blend="feather", bands=5):
        seen.update(feather=feather, blend=blend, bands=bands)
        M = np.stack([np.array([[1.0, 0, 10.0 * k], [0, 1.0, 0.5], [0, 0, 1.0]]) for k in range(3)])
        return dict(mosaic=torch.zeros(4, 6, 3, dtype=torch.uint8), mask=torch.zeros(4, 6, dtype=torch.uint8), M=M,
                    kept=np.array([True, False, True]), ref=1, H_pairs=np.stack([np.eye(3)] * 2), refine=None,
                    last_ms=dict(prep=1.0, forward=2.0, blend=3.0))

    class Event:
        def __init__(self, **kw):
            pass

        def record(self):
            pass

        def synchronize(self):
            pass

        def elapsed_time(self, other):
            return 0.5

    monkeypatch.setattr(mosaic, "build_mosaic", fake_build)
    monkeypatch.setattr(torch.cuda, "Event", Event)
    argv = ["--frames", str(raw), "--out_dir", str(tmp_path / "out")] + (["--blend", "multiband", "--bands", "7"] if blend == "multiband" else [])
    cli.run(cli.build_parser().parse_args(argv), None, lambda paths: None, lambda imgs: [b"jpeg"])
    txt = (tmp_path / "out" / "mosaic.txt").read_text().splitlines()
    assert seen == dict(feather=64, blend=blend, bands=7 if blend == "multiband" else 5)
    assert txt[0] == ("canvas 4 6 ref 1 blend multiband 7" if blend == "multiband" else "canvas 4 6 ref 1")
    assert txt[1] == "F_0.JPG kept 1 0 0 0 1 0.5 0 0 1" and txt[2].startswith("F_1.JPG dropped 1 0 10 ")
    assert (tmp_path / "out" / "mosaic.jpg").read_bytes() == b"jpeg"


# ---- the compiled kernels -----------------------------------------------------------------------------------------------
def _tool(name):
    p = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), name)
    return p if os.path.exists(p) else shutil.which(name)


NEEDS_TOOLKIT = pytest.mark.skipif(_tool("nvcc") is None or _tool("cuobjdump") is None, reason="the CUDA toolkit is not installed")
# sha256 of the SASS (instructions and encodings, one per line) of the warp and feathered-blend kernels as the parent of
# the multi-band blend compiled them with CUDA 12.9 (V12.9.86) and the library's flags
SASS_SHA256 = {"V12.9.86": {
    "_ZN3udh26warp_perspective_u8_kernelILi1EEEvPKhPKdiiPhiii": "4cf086833dca9fb1541e6ce6be759ab5dd46f95819f7b0a32bd20acbfd61752e",
    "_ZN3udh26warp_perspective_u8_kernelILi3EEEvPKhPKdiiPhiii": "6b66c89805d0a06eb07c220cac82937d435e41fde36bd4b1366552b15add20bf",
    "_ZN3udh22mosaic_blend_u8_kernelILi1ELb0ELb0ELb0EEEvPKNS_11MosaicFrameEiPKiS5_iiiiPhS6_PKdPKNS_8SeamMaskEPKNS_10GainMapDevE":
        "21efaa682281ae1163e2b5ece1ae58cdbca4af2f9fc5977050081a14a84a8136",
    "_ZN3udh22mosaic_blend_u8_kernelILi3ELb0ELb0ELb0EEEvPKNS_11MosaicFrameEiPKiS5_iiiiPhS6_PKdPKNS_8SeamMaskEPKNS_10GainMapDevE":
        "78dc2a9572571dea4c17fbebed4415bbafd4a50d6313609f0b6852dcfde96f59"}}


@pytest.fixture(scope="module")
def warp_object(tmp_path_factory):
    from unsuperviseddeephomographyral2018_b200 import build_ext
    obj = str(tmp_path_factory.mktemp("wp") / "warp_perspective.o")
    cmd = [_tool("nvcc")] + build_ext.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build_ext.CSRC, "warp_perspective.cu"),
                                                    "-o", obj]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, p.stdout
    return obj, p.stdout


@NEEDS_TOOLKIT
def test_warp_perspective_kernels_do_not_spill(warp_object):
    seen, current = {}, None
    for line in warp_object[1].splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            seen[current] = tuple(int(v) for v in m.groups())
    mb = [k for k in seen if "multiband_" in k]
    assert len(mb) == 6, mb                                       # base (plain, gain map), pyrDown, accumulate, collapse (level > 0, 0)
    assert len(seen) == 31, sorted(seen)                          # every entry function in warp_perspective.cu
    assert all(v == (0, 0, 0) for v in seen.values()), seen


@NEEDS_TOOLKIT
def test_warp_and_plain_blend_sass_is_unchanged(warp_object):
    ver = re.search(r"V\d+\.\d+\.\d+", subprocess.run([_tool("nvcc"), "--version"], stdout=subprocess.PIPE, text=True).stdout)
    if not ver or ver.group(0) not in SASS_SHA256:
        pytest.skip("the reference digest was taken with another nvcc (%s)" % (ver.group(0) if ver else "unknown"))
    for fn, want in SASS_SHA256[ver.group(0)].items():
        sass = subprocess.run([_tool("cuobjdump"), "-sass", "-fun", fn, warp_object[0]], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True, timeout=300)
        assert sass.returncode == 0, sass.stdout
        lines = [ln.strip() for ln in sass.stdout.splitlines() if re.match(r"\s+/\*([0-9a-f]{4,}\*/| 0x[0-9a-f]{16} \*/)", ln)]
        assert len(lines) > 1000, sass.stdout[:2000]
        assert hashlib.sha256("\n".join(lines).encode()).hexdigest() == want, fn
