"""Host-side tests of the sequence mosaic: chaining pair homographies to a reference frame, the canvas layout, the kernel's
candidate tile lists against a brute-force validity map, the blend rule's restatement oracle/mosaic.py, mosaic_images.py's
options and frame lists, and the compiled blend kernel (no spills; the warp kernel's SASS unchanged)."""
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


def T(dx, dy):
    return np.array([[1.0, 0, dx], [0, 1.0, dy], [0, 0, 1.0]])


def apply(G, pts):
    p = np.c_[pts, np.ones(len(pts))] @ G.T
    return p[:, :2] / p[:, 2:]


# ---- chaining ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_chain_equals_the_true_frame_to_reference_maps(where):
    from unsuperviseddeephomographyral2018_b200 import mosaic
    n = 7
    A, _ = SW.sweep_cameras(n, 480, 640, seed=3)
    H = SW.true_pairs(A)
    ref = {"first": 0, "middle": None, "last": n - 1}[where]
    G, r = mosaic.chain_to_reference(H, ref)
    assert r == {"first": 0, "middle": n // 2, "last": n - 1}[where]
    assert np.array_equal(G[r], np.eye(3))
    for k in range(n):
        true = np.linalg.inv(A[r]) @ A[k]
        true /= true[2, 2]
        assert G[k][2, 2] == 1.0
        assert np.abs(G[k] - true).max() <= 1e-9 * np.abs(true).max(), k
    assert mosaic.chain_to_reference(H, -1)[1] == n // 2


def test_chain_keeps_aligns_direction():
    """H_k takes frame k to frame k + 1 (align's image 1 -> image 2): a point of frame 0 chained to frame 2 lands where
    H_1 H_0 takes it, and frame 3's point comes back through inv(H_2)."""
    from unsuperviseddeephomographyral2018_b200 import mosaic
    H = np.stack([T(-100.0, 5.0), T(-80.0, -2.0), T(-90.0, 1.0)])       # the camera pans right: content moves left
    G, r = mosaic.chain_to_reference(H, 2)
    assert np.allclose(apply(G[0], np.array([[300.0, 50.0]])), [[120.0, 53.0]])
    assert np.allclose(apply(G[3], np.array([[10.0, 10.0]])), [[100.0, 9.0]])
    with pytest.raises(ValueError):
        mosaic.chain_to_reference(H, 4)


# ---- canvas ------------------------------------------------------------------------------------------------------------
def test_canvas_hand_worked():
    from unsuperviseddeephomographyral2018_b200 import mosaic
    sizes = [(10, 20), (10, 20)]
    # translation only: x 0..19 and 15..34, y 0..9 and 3..12
    M, (Hc, Wc), kept = mosaic.canvas(sizes, np.stack([np.eye(3), T(15, 3)]), 0)
    assert (Hc, Wc) == (13, 35) and kept.all() and np.array_equal(M[1], T(15, 3)) and np.array_equal(M[0], np.eye(3))
    # a 2x scale: x 0..38, y 0..18
    M, (Hc, Wc), _ = mosaic.canvas(sizes, np.stack([np.eye(3), np.diag([2.0, 2.0, 1.0])]), 0)
    assert (Hc, Wc) == (19, 39)
    # a negative offset: x0 = floor(-5.5) = -6, y0 = floor(-2.25) = -3
    M, (Hc, Wc), _ = mosaic.canvas(sizes, np.stack([np.eye(3), T(-5.5, -2.25)]), 0)
    assert (Hc, Wc) == (13, 26)
    assert np.array_equal(M[0], T(6, 3)) and np.array_equal(M[1], T(0.5, 0.75))


def test_canvas_drops_a_frame_behind_the_camera():
    from unsuperviseddeephomographyral2018_b200 import mosaic
    sizes = [(10, 20)] * 3
    # frame 2's grown corner x = w = 20 has denominator 1 - 0.05 * 20 = 0 (its pixel centres are all positive)
    P = np.array([[1.0, 0, 0], [0, 1.0, 0], [-0.05, 0, 1.0]])
    M, (Hc, Wc), kept = mosaic.canvas(sizes, np.stack([T(-10, 0), np.eye(3), P]), 1)
    assert kept.tolist() == [True, True, False] and (Hc, Wc) == (10, 30)
    # the reference frame is never dropped
    _, _, kept = mosaic.canvas(sizes[:2], np.stack([P, np.eye(3)]), 0)
    assert kept.tolist() == [True, True]


def test_canvas_limits_name_the_farthest_frame():
    from unsuperviseddeephomographyral2018_b200 import mosaic
    sizes = [(100, 200)] * 4
    G = np.stack([T(-150, 0), np.eye(3), T(150, 0), T(40000, 10)])
    with pytest.raises(ValueError, match="frame 3"):
        mosaic.canvas(sizes, G, 1)
    G[3] = T(300, 10)
    M, (Hc, Wc), _ = mosaic.canvas(sizes, G, 1)
    assert (Hc, Wc) == (110, 650)
    with pytest.raises(ValueError, match=r"110x650 canvas exceeds 70000 pixels; frame 3"):
        mosaic.canvas(sizes, G, 1, max_pixels=70000)
    G[0] = T(-600, 0)
    with pytest.raises(ValueError, match="frame 0"):
        mosaic.canvas(sizes, G, 1, max_pixels=70000)


# ---- the kernel's candidate lists ----------------------------------------------------------------------------------------
def _frames_for_lists(dh, dw):
    """(name, (h, w), M) of frames that reach a dh x dw canvas in different ways."""
    c, s = np.cos(0.7), np.sin(0.7)
    rot = T(dw / 2.0, dh / 2.0) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]]) @ T(-40, -30)
    persp = np.array([[1.2, 0.1, 30.0], [0.05, 0.9, 10.0], [2.5e-3, 1.5e-3, 1.0]])
    return [("shifted", (37, 53), T(-20.5, 13.25)),
            ("rotated", (60, 80), rot),
            ("magnified x8", (9, 11), T(5, 7) @ np.diag([8.0, 8.0, 1.0])),
            ("minified x1/8", (480, 640), T(100.25, 3.5) @ np.diag([0.125, 0.125, 1.0])),
            ("perspective", (90, 120), persp),
            ("horizon", (100, 100), np.array([[1.0, 0, 150.0], [0, 1.0, 20.0], [0, 0.0095, 1.0]])),
            ("outside", (20, 20), T(-100, -100)),
            ("singular", (30, 30), np.array([[1.0, 2.0, 3.0], [2.0, 4.0, 6.0], [0, 0, 1.0]]))]


@pytest.mark.parametrize("dh,dw", [(150, 333), (13, 200), (64, 64)])
def test_tile_lists_are_conservative(dh, dw):
    from oracle import mosaic as OM
    from unsuperviseddeephomographyral2018_b200 import _lib, ops
    frames = _frames_for_lists(dh, dw)
    ptr, idx = ops.mosaic_tile_lists(np.stack([m for _, _, m in frames]), [s for _, s, _ in frames], dh, dw)
    TH, TW = _lib.MOSAIC_TILE_H, _lib.MOSAIC_TILE_W
    gy, gx = -(-dh // TH), -(-dw // TW)
    assert ptr.dtype == np.int32 and idx.dtype == np.int32 and len(ptr) == gy * gx + 1 and ptr[0] == 0 and ptr[-1] == len(idx)
    listed = np.zeros((gy * gx, len(frames)), bool)
    for t in range(gy * gx):
        f = idx[ptr[t]:ptr[t + 1]]
        assert np.all(np.diff(f) > 0)                                   # frame order, no duplicates
        listed[t, f] = True
    for k, (name, (h, w), M) in enumerate(frames):
        valid, _ = OM.validity_weight(M, h, w, dh, dw, 1)
        pad = np.zeros((gy * TH, gx * TW), bool)
        pad[:dh, :dw] = valid
        need = pad.reshape(gy, TH, gx, TW).any(axis=(1, 3)).ravel()
        assert not np.any(need & ~listed[:, k]), name
        if name == "outside":
            assert not listed[:, k].any()
        if name in ("shifted", "magnified x8", "minified x1/8"):
            assert listed[:, k].sum() < gy * gx or gy * gx <= 4, name      # a bounding box, not every tile


# ---- the oracle ------------------------------------------------------------------------------------------------------------
def test_oracle_two_frames_hand_worked():
    """Two flat 4x4 frames (100 and 200), the second two columns right, on a 4x7 canvas with feather 1.  At column 2 frame
    A is 64/32 px from its edges in x (d = 32 on the inner rows) and frame B is on its edge (d = 0): (33 100 + 1 200 + 17) //
    34 = 103; column 3 mirrors it: (100 + 33 200 + 17) // 34 = 197.  The outer rows are on both frames' edges: weights
    1 and 1, (300 + 1) // 2 = 150.  Column 6 is outside both."""
    from oracle import mosaic as OM
    A, B = np.full((4, 4, 1), 100, np.uint8), np.full((4, 4, 1), 200, np.uint8)
    out, mask = OM.blend([A, B], np.stack([np.eye(3), T(2, 0)]), 4, 7, 1)
    edge, inner = [100, 100, 150, 150, 200, 200, 0], [100, 100, 103, 197, 200, 200, 0]
    assert out[..., 0].tolist() == [edge, inner, inner, edge]
    assert mask.tolist() == [[255] * 6 + [0]] * 4


def _random_frames(rng, C):
    frames = [rng.integers(0, 256, (h, w, C), np.uint8) for h, w in ((37, 53), (60, 45), (25, 90))]
    M = np.stack([T(3.5, 2.25) @ np.array([[0.9, 0.1, 0], [-0.08, 1.1, 0], [1e-3, 5e-4, 1.0]]), T(20, 10),
                  T(-10, 15) @ np.diag([1.3, 0.8, 1.0])])
    return frames, M


@pytest.mark.parametrize("C", [1, 3])
def test_oracle_feather_zero_is_the_rounded_plain_average(C):
    from oracle import mosaic as OM
    rng = np.random.default_rng(C)
    frames, M = _random_frames(rng, C)
    dh, dw = 70, 101
    out, mask = OM.blend(frames, M, dh, dw, 0)
    S = np.zeros((dh, dw, C), np.int64); n = np.zeros((dh, dw), np.int64)
    for F, Mk in zip(frames, M):
        valid, wt = OM.validity_weight(Mk, F.shape[0], F.shape[1], dh, dw, 0)
        assert np.all(wt[valid] == 1)
        v = cv2.warpPerspective(F if C == 3 else F[..., 0], Mk, (dw, dh)).reshape(dh, dw, C).astype(np.int64)
        S += v * valid[..., None]; n += valid
    assert n.max() == 3 and (n == 0).any()
    ref = np.where(n[..., None] > 0, (S + (n >> 1)[..., None]) // np.maximum(n, 1)[..., None], 0)
    assert np.array_equal(out, ref.astype(np.uint8)) and np.array_equal(mask, np.where(n > 0, 255, 0))


@pytest.mark.parametrize("feather", [0, 1, 64])
def test_oracle_single_frame_is_warp_perspective_where_valid(feather):
    from oracle import mosaic as OM
    rng = np.random.default_rng(feather)
    frames, M = _random_frames(rng, 3)
    out, mask = OM.blend(frames[:1], M[:1], 70, 101, feather)
    valid, _ = OM.validity_weight(M[0], 37, 53, 70, 101, feather)
    ref = cv2.warpPerspective(frames[0], M[0], (101, 70))
    assert np.array_equal(out, np.where(valid[..., None], ref, 0)) and np.array_equal(mask == 255, valid)
    assert 0 < valid.sum() < valid.size


def test_oracle_denominator_zero_is_invalid():
    """A zero denominator lands on source pixel (0, 0) (X = Y = 0, which is inside the frame): validity needs W != 0."""
    from oracle import mosaic as OM, warp_perspective as WP
    M = np.array([[1.0, 0, 0], [0, 1.0, 0], [0.125, 0, -1.0]])             # its own inverse: W = x / 8 - 1, 0 at x = 8
    X, Y = WP.source_coords(M, 4, 16)
    W = OM.denominator(M, 4, 16)
    z = W == 0
    assert z.any() and np.all(X[z] == 0) and np.all(Y[z] == 0)
    valid, _ = OM.validity_weight(M, 20, 20, 4, 16, 8)
    assert not valid[z].any()


# ---- the CLI ---------------------------------------------------------------------------------------------------------------
def test_cli_flags_and_defaults():
    import mosaic_images as cli
    a = cli.build_parser().parse_args(["--frames", "raw"])
    assert (a.glob, a.ref_frame, a.feather, a.out_dir) == ("*.JPG", -1, 64, "mosaic")
    assert (a.img_h, a.img_w, a.patch_size, a.numeric, a.batch_size, a.seed, a.model_name, a.loss_type, a.seeded_weights) == \
        (240, 320, 128, "bf16x3", 128, 0, "model.ckpt", "l1_loss", False)
    assert (a.refine_levels, a.refine_iters, a.refine_eps, a.refine_max_side) == (0, 50, 1e-6, None)
    a = cli.build_parser().parse_args(["--frames", "f.txt", "--ref_frame", "3", "--feather", "0", "--refine_levels", "-1",
                                       "--seeded_weights", "True", "--img_h", "142", "--img_w", "190"])
    assert (a.ref_frame, a.feather, a.refine_levels, a.seeded_weights, a.img_h, a.img_w) == (3, 0, -1, True, 142, 190)
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args([])


def test_align_images_options_unchanged():
    """align_images.py's parser shares its model options with mosaic_images.py; its options, order and defaults stay."""
    import align_images as cli
    p = cli.build_parser()
    assert [a.dest for a in p._actions] == ["help", "pairs", "img1", "img2", "model_dir", "model_name", "loss_type", "img_h",
                                            "img_w", "patch_size", "numeric", "batch_size", "out_dir", "save_warped",
                                            "seeded_weights", "seed", "refine_levels", "refine_iters", "refine_eps",
                                            "refine_max_side"]
    a = vars(p.parse_args([]))
    a.pop("model_dir")
    assert a == dict(pairs=None, img1=None, img2=None, model_name="model.ckpt", loss_type="l1_loss", img_h=240, img_w=320,
                     patch_size=128, numeric="bf16x3", batch_size=128, out_dir="aligned", save_warped=True, seeded_weights=False,
                     seed=0, refine_levels=0, refine_iters=50, refine_eps=1e-6, refine_max_side=None)


def test_cli_frame_lists(tmp_path):
    import mosaic_images as cli
    d = tmp_path / "raw"
    d.mkdir()
    for nm in ("DSC_0003.JPG", "DSC_0001.JPG", "DSC_0002.JPG", "notes.txt", "y.jpg", "x.jpg"):
        (d / nm).write_bytes(b"")
    names, paths = cli.frame_list(cli.build_parser().parse_args(["--frames", str(d)]))
    assert names == ["DSC_0001.JPG", "DSC_0002.JPG", "DSC_0003.JPG"] and paths[0] == str(d / "DSC_0001.JPG")
    names, _ = cli.frame_list(cli.build_parser().parse_args(["--frames", str(d), "--glob", "*.jpg"]))
    assert names == ["x.jpg", "y.jpg"]
    (tmp_path / "sub").mkdir()
    lst = tmp_path / "sub" / "frames.txt"
    lst.write_text("../raw/DSC_0002.JPG\n\n  b.png \na/c.jpg\n")
    names, paths = cli.frame_list(cli.build_parser().parse_args(["--frames", str(lst)]))
    assert names == ["../raw/DSC_0002.JPG", "b.png", "a/c.jpg"]
    assert paths == [os.path.join(str(tmp_path / "sub"), nm) for nm in names]
    lst.write_text("only.jpg\n")
    with pytest.raises(SystemExit):
        cli.frame_list(cli.build_parser().parse_args(["--frames", str(lst)]))


# ---- the compiled kernels -----------------------------------------------------------------------------------------------
def _tool(name):
    p = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), name)
    return p if os.path.exists(p) else shutil.which(name)


NEEDS_TOOLKIT = pytest.mark.skipif(_tool("nvcc") is None or _tool("cuobjdump") is None, reason="the CUDA toolkit is not installed")
# sha256 of warp_perspective_u8_kernel's SASS (instructions and encodings, one per line) as the parent of the mosaic kernel
# compiled it with CUDA 12.9 (V12.9.86) and the library's flags
WARP_SASS_SHA256 = {"V12.9.86": {
    "_ZN3udh26warp_perspective_u8_kernelILi1EEEvPKhPKdiiPhiii": "4cf086833dca9fb1541e6ce6be759ab5dd46f95819f7b0a32bd20acbfd61752e",
    "_ZN3udh26warp_perspective_u8_kernelILi3EEEvPKhPKdiiPhiii": "6b66c89805d0a06eb07c220cac82937d435e41fde36bd4b1366552b15add20bf"}}


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
def test_feathered_blend_instantiations_do_not_spill(warp_object):
    seen, current = {}, None
    for line in warp_object[1].splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current and "mosaic_" in current:
            seen[current] = tuple(int(v) for v in m.groups())
    assert len(seen) == 12, seen                                  # the blend: C = 1 and 3, plain, gains, masks, maps and combinations
    assert all(v == (0, 0, 0) for v in seen.values()), seen


@NEEDS_TOOLKIT
def test_warp_kernel_sass_is_unchanged(warp_object):
    ver = re.search(r"V\d+\.\d+\.\d+", subprocess.run([_tool("nvcc"), "--version"], stdout=subprocess.PIPE, text=True).stdout)
    if not ver or ver.group(0) not in WARP_SASS_SHA256:
        pytest.skip("the reference digest was taken with another nvcc (%s)" % (ver.group(0) if ver else "unknown"))
    for fn, want in WARP_SASS_SHA256[ver.group(0)].items():
        sass = subprocess.run([_tool("cuobjdump"), "-sass", "-fun", fn, warp_object[0]], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True, timeout=300)
        assert sass.returncode == 0, sass.stdout
        lines = [ln.strip() for ln in sass.stdout.splitlines() if re.match(r"\s+/\*([0-9a-f]{4,}\*/| 0x[0-9a-f]{16} \*/)", ln)]
        assert len(lines) > 1000, sass.stdout[:2000]
        assert hashlib.sha256("\n".join(lines).encode()).hexdigest() == want, fn
