"""Host-side tests of seams found at a reduced resolution (oracle/seam_scale.py): the INTER_LINEAR_EXACT restatement and the
library's tap tables against cv2.resize byte for byte (both forms, ties included), the oracle at a = 1 against the
full-resolution blend masks, the megapix -> scale rule and the seam geometry, the graded multi-band feed against cv2's
blender, mosaic_images.py's --seam_megapix and mosaic.txt, the C ABI's argument checks, and the compiled kernels."""
import ctypes
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_seam_gc_logic as GL  # noqa: E402
import test_seam_logic as SL  # noqa: E402

cv2 = pytest.importorskip("cv2")
from oracle import multiband as MB  # noqa: E402
from oracle import seam as SM  # noqa: E402
from oracle import seam_gc as GC  # noqa: E402
from oracle import seam_scale as SS  # noqa: E402

EXACT = cv2.INTER_LINEAR_EXACT


def _img(rng, h, w, C):
    return rng.integers(0, 256, (h, w, C) if C == 3 else (h, w), np.uint8)


def resize_cases():
    """(h, w, C, form, args): 240 random cases in both forms, then the edges."""
    rng = np.random.default_rng(5)
    out = []
    for t in range(240):
        C = (1, 3)[t % 2]
        h, w = (int(v) for v in rng.integers(1, 260, 2))
        if t % 2 == 0:
            a = float(rng.uniform(0.09, 4.3))
            if SS.fx_size(h, a) >= 1 and SS.fx_size(w, a) >= 1:
                out.append((h, w, C, "fx", a))
        else:
            out.append((h, w, C, "dsize", (int(rng.integers(1, 400)), int(rng.integers(1, 400)))))
    for C in (1, 3):
        out += [(1, 1, C, "dsize", (5, 7)), (1, 9, C, "dsize", (3, 1)), (9, 1, C, "fx", 2.5), (5, 300, C, "fx", 0.2),
                (37, 53, C, "fx", 1.0), (37, 53, C, "dsize", (37, 53)), (64, 96, C, "fx", 0.5), (65, 97, C, "fx", 0.5),
                (20, 30, C, "fx", 12.0), (7, 11, C, "dsize", (84, 132)), (3000, 40, C, "fx", 0.0913),
                (1080, 1920, C, "fx", 0.21957751641341997), (89, 110, C, "fx", 0.9965875624784407)]
    return out


CASES = resize_cases()


@pytest.mark.parametrize("h,w,C,form,arg", CASES, ids=["%dx%dx%d-%s-%s" % (h, w, C, f, a) for h, w, C, f, a in CASES])
def test_restatement_equals_cv2(h, w, C, form, arg):
    img = _img(np.random.default_rng(h * 7 + w), h, w, C)
    if form == "fx":
        ref, got = cv2.resize(img, None, fx=arg, fy=arg, interpolation=EXACT), SS.resize_exact(img, fx=arg)
    else:
        ref, got = cv2.resize(img, (arg[1], arg[0]), interpolation=EXACT), SS.resize_exact(img, arg[0], arg[1])
    assert got.shape == ref.shape and np.array_equal(got, ref)


@pytest.mark.parametrize("h,w", [(2, 2), (3, 5), (1, 4)])
def test_ties_round_to_even(h, w):
    """x256 upscales put (f - s) 256 on k + 1/2 at every output: cv2 rounds those weights to even."""
    c1 = SS.exact_axis(w, 256 * w, 1.0 / 256.0)[2]
    f = (np.arange(256 * w) + 0.5) / 256.0 - 0.5
    frac = (f - np.floor(f)) * 256.0
    assert np.all(frac - np.floor(frac) == 0.5)
    assert np.array_equal(c1, np.rint(frac).astype(np.int64)) and not np.array_equal(c1, np.floor(frac + 0.5).astype(np.int64))
    img = _img(np.random.default_rng(h + w), h, w, 3)
    assert np.array_equal(SS.resize_exact(img, 256 * h, 256 * w), cv2.resize(img, (256 * w, 256 * h), interpolation=EXACT))
    assert np.array_equal(SS.resize_exact(img, fx=256.0), cv2.resize(img, None, fx=256.0, fy=256.0, interpolation=EXACT))


def test_fx_and_dsize_forms_differ():
    """cv2's two forms sample with different scales: on a 1080 x 1920 frame at a = 0.2196 they differ in most bytes."""
    img = _img(np.random.default_rng(1), 1080, 1920, 3)
    a = 0.2196
    fx = cv2.resize(img, None, fx=a, fy=a, interpolation=EXACT)
    ds = cv2.resize(img, (fx.shape[1], fx.shape[0]), interpolation=EXACT)
    assert (fx != ds).mean() > 0.5
    assert np.array_equal(SS.resize_exact(img, fx=a), fx)


@pytest.mark.parametrize("h,w,C,form,arg", CASES[::7])
def test_library_table_equals_the_restatement(h, w, C, form, arg):
    from unsuperviseddeephomographyral2018_b200 import ops
    if form == "fx":
        dh, dw, ix, iy, scale = SS.fx_size(h, arg), SS.fx_size(w, arg), arg, arg, arg
    else:
        dh, dw, ix, iy, scale = arg[0], arg[1], arg[1] / float(w), arg[0] / float(h), None
    if (dh, dw) == (h, w):
        ix = iy = 1.0
    want = np.concatenate([np.concatenate(SS.exact_axis(w, dw, 1.0 / ix)), np.concatenate(SS.exact_axis(h, dh, 1.0 / iy))])
    assert np.array_equal(ops.linear_exact_table(h, w, dh, dw, scale), want.astype(np.int32))


# ---- the scale and the geometry -------------------------------------------------------------------------------------------
def test_megapix_rule():
    from unsuperviseddeephomographyral2018_b200 import mosaic
    assert mosaic.seam_scale([(1080, 1920), (4000, 3000)], 0.1) == SS.seam_scale([(1080, 1920)], 0.1) == math.sqrt(0.1e6 / (1080 * 1920))
    assert mosaic.seam_scale([(480, 640), (10, 10)], 0.6) == 1.0                   # clamped at 1; the first frame counts
    assert mosaic.seam_scale([(3000, 4000)], 0.1) == pytest.approx(0.0912870929)
    with pytest.raises(ValueError):
        mosaic.seam_scale([(10, 10)], 0)


def test_seam_geometry():
    from unsuperviseddeephomographyral2018_b200 import mosaic
    frames, M, (Hc, Wc) = SL.frame_case("warped")
    a = 0.37
    sizes = [f.shape[:2] for f in frames]
    Ms, small, canvas = mosaic.seam_geometry(M, sizes, Hc, Wc, a)
    Mo, small_o, canvas_o = SS.seam_geometry(M, sizes, Hc, Wc, a)
    assert np.array_equal(Ms, Mo) and small == small_o and canvas == canvas_o == (math.ceil(a * Hc), math.ceil(a * Wc))
    C = SS.centre_map(a)
    for Mk, Msk in zip(M, Ms):
        assert np.allclose(Msk, C @ Mk @ np.linalg.inv(C), rtol=0, atol=1e-12)
    # C(a) is the resize's own map: the resize samples its output pixel d at the source position C(a)^-1 d
    ramp = np.tile(np.arange(0, 250, 10, dtype=np.uint8), (3, 1))                 # 3 x 25, linear in x
    out = cv2.resize(ramp, None, fx=0.4, fy=0.4, interpolation=EXACT)
    xs = (np.linalg.inv(SS.centre_map(0.4)) @ np.stack([np.arange(out.shape[1]), np.zeros(out.shape[1]), np.ones(out.shape[1])]))[0]
    inside = (xs >= 0) & (xs <= 24)
    assert np.all(np.abs(out[0, inside] - 10 * xs[inside]) <= 0.5 + 10 / 256)
    with pytest.raises(ValueError, match="empty at seam scale"):
        mosaic.seam_geometry(M, [(1, 1)] + sizes[1:], Hc, Wc, 0.1)


@pytest.mark.parametrize("finder,name", [("voronoi", "warped"), ("voronoi", "clipped"), ("voronoi", "sweep"), ("gc_color", "order"),
                                         ("gc_color", "warped")])
def test_oracle_at_scale_one_is_the_full_resolution_rule(finder, name):
    """The scaled rule run at a = 1 (identity resize and geometry, every tap weight 0) gives oracle/seam's blend masks."""
    frames, M, (Hc, Wc) = GL.gc_case(name) if finder == "gc_color" else SL.frame_case(name)
    take, bm, _ = SS.masks(frames, M, Hc, Wc, 1.0, finder)
    t, imgs, masks, tls = SM.fed(frames, M, Hc, Wc)
    seams = GC.restate(imgs, masks, tls)[0] if finder == "gc_color" else SM.restate(masks, tls)
    assert take == t and SL._equal(bm, SM.blend_masks(seams, masks))


def test_scaled_masks_are_graded_and_inside_the_validity():
    frames, M, (Hc, Wc) = SL.frame_case("sweep")
    take, bm, (take_s, seams, rois_s, canvas_s) = SS.masks(frames, M, Hc, Wc, 0.3)
    _, _, masks, _ = SM.fed(frames, M, Hc, Wc)
    vals = np.unique(np.concatenate([b.ravel() for b in bm]))
    assert vals[0] == 0 and vals[-1] == 255 and len(vals) > 10
    assert all(not np.any(b[m == 0]) for b, m in zip(bm, masks))


# ---- the graded multi-band feed ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bands", [0, 3, 5])
def test_graded_multiband_feed_equals_cv2(bands):
    frames, M, (Hc, Wc) = SL.frame_case("sweep")
    take, bm, _ = SS.masks(frames, M, Hc, Wc, 0.25)
    _, imgs, _, tls = SM.fed(frames, M, Hc, Wc)
    ref, ref_mask, dst = MB.cv2_blend(imgs, bm, tls, Hc, Wc, bands)
    got = MB.restate(imgs, bm, tls, Hc, Wc, bands)
    assert np.array_equal(got["dst"], dst) and np.array_equal(got["mask"], ref_mask) and np.array_equal(got["mosaic"], ref)


# ---- the CLI ----------------------------------------------------------------------------------------------------------------------
def test_cli_seam_megapix_flag():
    import mosaic_images as cli
    assert cli.build_parser().parse_args(["--frames", "raw"]).seam_megapix == -1
    assert cli.build_parser().parse_args(["--frames", "raw", "--seam", "gc_color", "--seam_megapix", "0.1"]).seam_megapix == 0.1
    args = cli.build_parser().parse_args(["--frames", "raw", "--seam_megapix", "0.1"])
    with pytest.raises(SystemExit, match="needs --seam"):
        cli.run(args, None, None, None)


@pytest.mark.parametrize("megapix,scale", [(None, 1.0), (0.1, 0.21957751641341997), (5.0, 1.0)])
def test_cli_mosaic_txt(tmp_path, monkeypatch, megapix, scale):
    """With --seam_megapix giving a < 1 the first line ends in ` seam FINDER A` ('%.17g'); otherwise it is unchanged."""
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
                    kept=np.array([True, True, True]), ref=1, H_pairs=np.stack([np.eye(3)] * 2), refine=None,
                    gains=np.ones((3, 3)), seam_scale=scale, last_ms=dict(prep=1.0, forward=2.0, blend=3.0, seam=0.25))

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
    argv = ["--frames", str(raw), "--out_dir", str(tmp_path / "out"), "--seam", "gc_color"]
    if megapix is not None:
        argv += ["--seam_megapix", str(megapix)]
    cli.run(cli.build_parser().parse_args(argv), None, lambda paths: None, lambda imgs: [b"jpeg"])
    txt = (tmp_path / "out" / "mosaic.txt").read_text().splitlines()
    assert seen == (dict(seam="gc_color") if megapix is None else dict(seam="gc_color", seam_megapix=megapix))
    assert txt[0] == "canvas 4 6 ref 1 seam gc_color" + (" %.17g" % scale if scale < 1 else "")
    if scale < 1:
        assert float(txt[0].split()[-1]) == scale


def test_build_mosaic_needs_a_finder_for_seam_megapix():
    from unsuperviseddeephomographyral2018_b200 import mosaic

    class Est:
        last_ms = {}

        def estimate(self, a, b):
            return np.stack([np.eye(3)] * len(a)), None, None

    class F:
        shape = (10, 10, 3)

    with pytest.raises(ValueError, match="seam_megapix"):
        mosaic.build_mosaic(Est(), [F(), F()], seam_megapix=0.1, max_pixels=10 ** 6)


# ---- the C ABI ---------------------------------------------------------------------------------------------------------------------
def test_entries_reject_bad_arguments_before_touching_the_device():
    from unsuperviseddeephomographyral2018_b200 import _lib
    L = _lib.lib
    p = ctypes.c_void_p(256)                          # never dereferenced: every call below fails its argument checks
    for a, msg in (((None, p, p, 1, 4, 4, 3, 2, 2), b"null pointer"), ((p, p, p, 1, 4, 4, 2, 2, 2), b"channels must be 1 or 3"),
                   ((p, p, p, -1, 4, 4, 3, 2, 2), b"bad dimensions"), ((p, p, p, 1, 4, 4, 3, 0, 2), b"bad dimensions"),
                   ((p, p, p, 1, 4, 4, 3, 65536, 65536), b"bad dimensions")):
        assert L.udh_resize_linear_exact_u8(*a, None) == _lib.EINVAL, a
        assert b"udh_resize_linear_exact_u8: " + msg in L.udh_last_error()
    n = 2
    frames = (ctypes.c_void_p * n)(256, 512)
    seams = (ctypes.c_void_p * n)(256, None)
    sizes = (ctypes.c_int32 * (2 * n))(4, 4, 4, 4)
    rois = (ctypes.c_int32 * (4 * n))(0, 0, 8, 8, 4, 4, 12, 12)
    srois = (ctypes.c_int32 * (4 * n))(0, 0, 3, 3, 0, 0, 0, 0)
    srois_null = (ctypes.c_int32 * (4 * n))(0, 0, 3, 3, 1, 1, 3, 3)
    srois_out = (ctypes.c_int32 * (4 * n))(0, 0, 3, 3, 1, 1, 5, 3)
    nb = L.udh_mosaic_seam_upscale_workspace_bytes(rois, srois, n, 4, 4, 0.3, 12, 12)
    assert nb > 0
    assert L.udh_mosaic_seam_upscale_workspace_bytes(rois, srois, n, 4, 4, 1.5, 12, 12) == 0
    up = lambda fr, sr, sh, sw, a, ws: L.udh_mosaic_seam_upscale_u8(fr, sizes, p, rois, seams, sr, n, sh, sw, a, 12, 12, p, p, ws, None)
    for args, msg in (((None, srois, 4, 4, 0.3, nb), b"null pointer"), ((frames, srois, 4, 4, 0.0, nb), b"scale must be in (0, 1]"),
                      ((frames, srois, 4, 4, 1.01, nb), b"scale must be in (0, 1]"), ((frames, srois, 13, 4, 0.3, nb), b"bad dimensions"),
                      ((frames, srois_null, 4, 4, 0.3, nb), b"frame 1's seam mask is a null pointer"),
                      ((frames, srois_out, 4, 4, 0.3, nb), b"frame 1's seam ROI (1, 1)..(5, 3) leaves the 4x4 seam canvas")):
        assert up(*args) == _lib.EINVAL, msg
        assert b"udh_mosaic_seam_upscale_u8: " + msg in L.udh_last_error(), L.udh_last_error()
    assert up(frames, srois, 4, 4, 0.3, nb - 1) == _lib.EWS
    assert b"udh_mosaic_seam_upscale_u8: workspace of" in L.udh_last_error()


# ---- the compiled kernels ---------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(SL._tool("nvcc") is None, reason="the CUDA toolkit is not installed")
def test_seam_scale_kernels_do_not_spill(tmp_path):
    from unsuperviseddeephomographyral2018_b200 import build_ext
    cmd = [SL._tool("nvcc")] + build_ext.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build_ext.CSRC, "seam_scale.cu"),
                                                       "-o", str(tmp_path / "ss.o")]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, p.stdout
    seen, current = {}, None
    for line in p.stdout.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            seen[current] = tuple(int(v) for v in m.groups())
    # the resize (C = 1 and 3), the dilation and the upscale
    assert len(seen) == 4, seen
    assert all(v == (0, 0, 0) for v in seen.values()), seen
