"""Host-side tests of the mosaic's seams: the NumPy restatement (oracle/seam.py) against cv2.detail's Voronoi seam finder
byte for byte on every kind of pair, the blend masks against cv2.dilate + bitwise_and, the end-to-end multi-band
reference against cv2's blender fed cv2's seams, the pair lists, mosaic_images.py's --seam and mosaic.txt, and the
compiled kernels (no spills)."""
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
from oracle import multiband as MB  # noqa: E402
from oracle import seam as SM  # noqa: E402


def T(dx, dy):
    return np.array([[1.0, 0, dx], [0, 1.0, dy], [0, 0, 1.0]])


def full(h, w):
    return np.full((h, w), 255, np.uint8)


# ---- the cases, shared with tests/test_gpu_seam.py ----------------------------------------------------------------------
def mask_case(name):
    """(masks, tls) of a named hand-built case."""
    if name == "tie":                                          # an overlap 7 px wide: its middle column is a tie
        return [full(20, 30), full(20, 30)], [(0, 0), (23, 0)]
    if name == "order":                                        # three frames, each overlapping both others
        return [full(30, 40), full(30, 40), full(30, 40)], [(0, 0), (25, 6), (10, 22)]
    if name == "contained":                                    # frame 1 inside frame 0, frame 2 inside frame 1
        return [full(40, 50), full(20, 24), full(6, 6)], [(0, 0), (12, 9), (20, 15)]
    if name == "no_unique":                                    # identical ROIs and masks: no pixel is either frame's alone
        m = full(12, 15)
        m[0, :] = 0
        return [m, m.copy()], [(3, 4), (3, 4)]
    if name == "holes":                                        # sparse masks: windows where one frame has no unique pixel
        rng = np.random.default_rng(3)
        ms = [np.where(rng.random((25, 25)) < 0.08, 255, 0).astype(np.uint8) for _ in range(4)]
        return ms, [(0, 0), (14, 2), (5, 15), (30, 30)]
    raise KeyError(name)


def frame_case(name):
    """(frames uint8 RGB, M [n,3,3] frame -> canvas, (Hc, Wc)) of a named case of warped frames."""
    rng = np.random.default_rng(sum(map(ord, name)))
    c, s = np.cos(0.4), np.sin(0.4)
    rot = T(60, 20) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])
    persp = np.array([[0.9, 0.05, 80.0], [-0.03, 1.05, -10.0], [4e-4, -2e-4, 1.0]])
    if name == "clipped":                                      # ROIs clipped at every edge of the canvas
        sizes, M, canvas = [(40, 60), (40, 60), (30, 30)], [T(-12.5, -7.25), T(30, 9.5), T(-5, 20)], (45, 80)
    elif name == "warped":                                     # rotation and perspective: non-rectangular masks
        sizes, M, canvas = [(120, 160), (100, 140), (90, 120)], [T(5.5, 3.25), rot, persp @ T(-20, 30)], (220, 280)
    elif name == "stacked":                                    # 20 frames within a few pixels of each other: 190 pairs
        sizes = [(24, 30)] * 20
        M, canvas = [T(2 + (k % 5) + 0.5 * (k % 2), 3 + (k % 3)) for k in range(20)], (33, 41)
    elif name == "sweep":
        _, frames, _, H = SW.sweep(4, 120, 160, seed=2)
        return _chain(frames, H)
    else:
        raise KeyError(name)
    frames = [rng.integers(0, 256, (h, w, 3), np.uint8) for h, w in sizes]
    return frames, np.stack(M), canvas


def _chain(frames, H):
    from unsuperviseddeephomographyral2018_b200 import mosaic
    G, ref = mosaic.chain_to_reference(H)
    M, (Hc, Wc), kept = mosaic.canvas([f.shape[:2] for f in frames], G, ref)
    assert kept.all()
    return frames, M, (Hc, Wc)


MASK_CASES = ["tie", "order", "contained", "no_unique", "holes"]
FRAME_CASES = ["clipped", "warped", "stacked", "sweep"]


def _equal(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


# ---- the rule against cv2 ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", MASK_CASES)
def test_restatement_equals_cv2_on_hand_built_pairs(name):
    masks, tls = mask_case(name)
    ref = SM.cv2_seams(masks, tls)
    assert _equal(SM.restate(masks, tls), ref)
    assert _equal(masks, mask_case(name)[0])                  # the inputs are left alone


@pytest.mark.parametrize("name", FRAME_CASES)
def test_restatement_equals_cv2_on_warped_frames(name):
    frames, M, (Hc, Wc) = frame_case(name)
    take, _, masks, tls = SM.fed(frames, M, Hc, Wc)
    ref = SM.cv2_seams(masks, tls)
    assert _equal(SM.restate(masks, tls), ref)
    if name == "stacked":
        assert len(SM.pairs(tls, [m.shape for m in masks])) == 190
    if name == "clipped":
        rois = [(x, y, x + m.shape[1], y + m.shape[0]) for (x, y), m in zip(tls, masks)]
        assert min(r[0] for r in rois) == 0 and min(r[1] for r in rois) == 0
        assert max(r[2] for r in rois) == Wc and max(r[3] for r in rois) == Hc
    if name == "warped":
        assert any((m == 0).any() for m in masks)             # corners outside the warped frames


def test_tie_goes_to_the_later_frame():
    masks, tls = mask_case("tie")
    s = SM.restate(masks, tls)
    # overlap x 23..29: columns 23..25 are nearer frame 0's own pixels, 27..29 frame 1's, 26 is equidistant
    assert (s[0][:, 23:26] == 255).all() and (s[0][:, 26:] == 0).all()
    assert (s[1][:, :3] == 0).all() and (s[1][:, 3:] == 255).all()                # canvas column 26 goes to frame 1
    a, b = [m.copy() for m in masks]
    SM.find_in_pair(a, b, tls[0], tls[1], (23, 0, 30, 20), tie_to_j=False)
    assert not np.array_equal(a, s[0])


def test_visiting_order_changes_the_result():
    masks, tls = mask_case("order")
    fwd = SM.restate(masks, tls)
    perm = [2, 0, 1]
    rev = SM.restate([masks[k] for k in perm], [tls[k] for k in perm])
    assert _equal(rev, SM.cv2_seams([masks[k] for k in perm], [tls[k] for k in perm]))
    back = [None] * 3
    for q, k in enumerate(perm):
        back[k] = rev[q]
    assert not _equal(back, fwd)


def test_contained_frames_vanish_and_empty_windows_clear_the_first_frame():
    s = SM.restate(*mask_case("contained"))
    assert (s[1] == 0).all() and (s[2] == 0).all() and (s[0] == 255).all()
    masks, tls = mask_case("no_unique")
    s = SM.restate(masks, tls)
    assert (s[0] == 0).all() and np.array_equal(s[1], masks[1])


def test_l1_distance_is_exact():
    rng = np.random.default_rng(0)
    for _ in range(20):
        src = rng.random((int(rng.integers(1, 30)), int(rng.integers(1, 30)))) < rng.uniform(0, 0.1)
        d = SM.l1_distance(src)
        ys, xs = np.nonzero(src)
        if not len(ys):
            assert (d == SM.INF).all()
            continue
        yy, xx = np.mgrid[:src.shape[0], :src.shape[1]]
        want = np.min(np.abs(yy[..., None] - ys) + np.abs(xx[..., None] - xs), -1)
        assert np.array_equal(d, want)


def test_distances_past_65536_are_not_capped():
    """Two full 2 x 140000 frames one column apart: each holds one column alone, 140000 px from the other's, so the seam
    falls at x = 70000, where both distances exceed 65536 (a cap there would tie them and move the seam)."""
    masks, tls = [full(2, 140000), full(2, 140000)], [(0, 0), (1, 0)]
    ref = SM.cv2_seams(masks, tls)
    assert _equal(SM.restate(masks, tls), ref)
    assert (ref[0][:, :70000] == 255).all() and (ref[0][:, 70000:] == 0).all()


# ---- the blend masks and the end-to-end reference ------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["warped", "sweep"])
def test_blend_masks_are_dilate_and_validity(name):
    frames, M, (Hc, Wc) = frame_case(name)
    _, _, masks, tls = SM.fed(frames, M, Hc, Wc)
    seams = SM.restate(masks, tls)
    got = SM.blend_masks(seams, masks)
    for s, m, g in zip(seams, masks, got):
        p = np.pad(s, 1)
        dil = np.zeros_like(s)
        for dy in range(3):
            for dx in range(3):
                dil = np.maximum(dil, p[dy:dy + s.shape[0], dx:dx + s.shape[1]])
        assert np.array_equal(g, np.where((dil != 0) & (m != 0), 255, 0).astype(np.uint8))
        assert np.array_equal(g, cv2.bitwise_and(cv2.dilate(s, np.ones((3, 3), np.uint8)), m))


@pytest.mark.parametrize("name", ["warped", "sweep"])
def test_multiband_reference_equals_cv2_fed_cv2_seams(name):
    frames, M, (Hc, Wc) = frame_case(name)
    take, imgs, masks, tls = SM.fed(frames, M, Hc, Wc)
    bm = SM.blend_masks(SM.cv2_seams(masks, tls), masks)
    ref = MB.restate(imgs, bm, tls, Hc, Wc, 5)
    out, mask = SM.multiband(frames, M, Hc, Wc, 5)
    assert np.array_equal(out, ref["mosaic"]) and np.array_equal(mask, ref["mask"])
    unseamed, _ = MB.blend(frames, M, Hc, Wc, 5)
    assert not np.array_equal(out, unseamed)


def test_roi_pairs_without_the_diagonal_are_cv2s_visiting_order():
    from unsuperviseddeephomographyral2018_b200 import ops
    rng = np.random.default_rng(5)
    for _ in range(20):
        m = int(rng.integers(1, 30))
        x0, y0 = rng.integers(0, 200, m), rng.integers(0, 200, m)
        rois = np.stack([x0, y0, x0 + rng.integers(1, 60, m), y0 + rng.integers(1, 60, m)], 1)
        ptr, pj = ops.roi_pairs(rois, False)
        got = [(i, int(j)) for i in range(m) for j in pj[ptr[i]:ptr[i + 1]]]
        assert got == [(i, j) for i, j, _ in SM.pairs([(int(a), int(b)) for a, b in rois[:, :2]],
                                                      [(int(r[3] - r[1]), int(r[2] - r[0])) for r in rois])]


# ---- the CLI ---------------------------------------------------------------------------------------------------------------
def test_cli_seam_flag():
    import mosaic_images as cli
    assert cli.build_parser().parse_args(["--frames", "raw"]).seam == "none"
    assert cli.build_parser().parse_args(["--frames", "raw", "--seam", "voronoi"]).seam == "voronoi"
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args(["--frames", "raw", "--seam", "graphcut"])


def test_build_mosaic_rejects_other_seams():
    from unsuperviseddeephomographyral2018_b200 import mosaic

    class Est:
        last_ms = {}

        def estimate(self, a, b):
            return np.stack([np.eye(3)] * len(a)), None, None

    class F:
        shape = (10, 10, 3)

    with pytest.raises(ValueError, match="seam"):
        mosaic.build_mosaic(Est(), [F(), F()], seam="graphcut", max_pixels=10 ** 6)


@pytest.mark.parametrize("seam", ["none", "voronoi"])
def test_cli_mosaic_txt(tmp_path, monkeypatch, seam):
    """Without --seam mosaic.txt and build_mosaic's arguments are the parent's; with it the first line ends in ` seam
    voronoi`, after the blend and compensation."""
    import torch
    import mosaic_images as cli
    from unsuperviseddeephomographyral2018_b200 import mosaic
    raw = tmp_path / "raw"
    raw.mkdir()
    for k in range(3):
        (raw / ("F_%d.JPG" % k)).write_bytes(b"")
    seen = {}

    def fake_build(est, imgs, ref, refine, feather, float32_M=False, blend="feather", bands=5, **kw):
        seen.update(kw)
        M = np.stack([np.array([[1.0, 0, 10.0 * k], [0, 1.0, 0.5], [0, 0, 1.0]]) for k in range(3)])
        return dict(mosaic=torch.zeros(4, 6, 3, dtype=torch.uint8), mask=torch.zeros(4, 6, dtype=torch.uint8), M=M,
                    kept=np.array([True, False, True]), ref=1, H_pairs=np.stack([np.eye(3)] * 2), refine=None,
                    gains=np.ones((3, 3)), last_ms=dict(prep=1.0, forward=2.0, blend=3.0, compensate=0.5, seam=0.25))

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
    argv = ["--frames", str(raw), "--out_dir", str(tmp_path / "out"), "--blend", "multiband", "--compensate", "gain"]
    if seam != "none":
        argv += ["--seam", seam]
    cli.run(cli.build_parser().parse_args(argv), None, lambda paths: None, lambda imgs: [b"jpeg"])
    txt = (tmp_path / "out" / "mosaic.txt").read_text().splitlines()
    if seam == "none":
        assert seen == dict(compensate="gain", compensate_feeds=1)
        assert txt[0] == "canvas 4 6 ref 1 blend multiband 5 compensate gain 1"
    else:
        assert seen == dict(compensate="gain", compensate_feeds=1, seam="voronoi")
        assert txt[0] == "canvas 4 6 ref 1 blend multiband 5 compensate gain 1 seam voronoi"
    assert txt[1].startswith("F_0.JPG kept 1 0 0 0 1 0.5 0 0 1 ")


# ---- the compiled kernels -----------------------------------------------------------------------------------------------
def _tool(name):
    p = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), name)
    return p if os.path.exists(p) else shutil.which(name)


@pytest.mark.skipif(_tool("nvcc") is None, reason="the CUDA toolkit is not installed")
def test_seam_and_masked_blend_kernels_do_not_spill(tmp_path):
    from unsuperviseddeephomographyral2018_b200 import build_ext
    cmd = [_tool("nvcc")] + build_ext.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build_ext.CSRC, "warp_perspective.cu"),
                                                    "-o", str(tmp_path / "wp.o")]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, p.stdout
    seen, current = {}, None
    for line in p.stdout.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current and re.search(r"seam_|mosaic_blend_u8_kernelILi\dELb[01]ELb1ELb0E|multiband_base_kernelILb0E", current):
            seen[current] = tuple(int(v) for v in m.groups())
    # validity, columns, rows, blend masks, the masked feathered blend (C = 1 and 3, with and without gains), the
    # multi-band base (which takes the masks)
    assert len(seen) == 9, seen
    assert all(v == (0, 0, 0) for v in seen.values()), seen
