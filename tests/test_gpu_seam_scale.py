"""GPU tests of seams found at a reduced resolution: udh_resize_linear_exact_u8 against cv2.resize(INTER_LINEAR_EXACT) byte
for byte (both forms, batches, 12 MP -> 0.1 MP), the seam-scale seams against cv2's Voronoi finder and the graph-cut
restatement, the graded full-resolution blend masks against oracle/seam_scale's upscale of the GPU's own seams, both
blends (with gains and with gain maps) against oracle/seam_scale, scale 1 against the full-resolution call, run
independence, the buffer contract, build_mosaic and mosaic_images.py --seam_megapix end to end, and the numbers the
feature reports (the pixels left without weight, a drifting sweep's score)."""
import os
import sys

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _buffer_contract as BC  # noqa: E402
import _mosaic_sweep as SW  # noqa: E402
import test_gpu_seam as GS  # noqa: E402
import test_seam_logic as SL  # noqa: E402
from oracle import seam as SM  # noqa: E402
from oracle import seam_gc as GC  # noqa: E402
from oracle import seam_scale as SS  # noqa: E402

pytestmark = pytest.mark.gpu
EXACT = cv2.INTER_LINEAR_EXACT
T = SL.T


def _ops():
    from unsuperviseddeephomographyral2018_b200 import ops
    return ops


def _mosaic():
    from unsuperviseddeephomographyral2018_b200 import mosaic
    return mosaic


# ---- the resize -----------------------------------------------------------------------------------------------------------------
RESIZES = [((1, 1), "fx", 3.0), ((5, 7), "dsize", (1, 13)), ((37, 53), "fx", 0.37), ((64, 96), "fx", 0.5), ((97, 130), "dsize", (33, 401)),
           ((2, 3), "fx", 256.0), ((120, 160), "fx", 12.0), ((1080, 1920), "fx", 0.21957751641341997), ((480, 640), "dsize", (480, 640)),
           ((89, 110), "fx", 0.9965875624784407)]


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("size,form,arg", RESIZES)
def test_resize_equals_cv2(size, form, arg, C):
    rng = np.random.default_rng(size[0] * 31 + size[1])
    src = rng.integers(0, 256, (3,) + size + (C,), np.uint8)
    s = torch.from_numpy(src).cuda()
    got = (_ops().resize_linear_exact_u8(s, scale=arg) if form == "fx" else _ops().resize_linear_exact_u8(s, arg[0], arg[1])).cpu().numpy()
    for k in range(3):
        img = src[k] if C == 3 else src[k, ..., 0]
        ref = cv2.resize(img, None, fx=arg, fy=arg, interpolation=EXACT) if form == "fx" else cv2.resize(img, arg[::-1], interpolation=EXACT)
        assert np.array_equal(got[k].reshape(ref.shape), ref), k
    one = _ops().resize_linear_exact_u8(s[1], scale=arg) if form == "fx" else _ops().resize_linear_exact_u8(s[1], arg[0], arg[1])
    assert np.array_equal(one.cpu().numpy(), got[1])


def test_resize_12mp_to_a_tenth_of_a_megapixel():
    img = SW.texture(np.random.default_rng(12), 3000, 4000)
    a = _mosaic().seam_scale([(3000, 4000)], 0.1)
    got = _ops().resize_linear_exact_u8(torch.from_numpy(img).cuda(), scale=a).cpu().numpy()
    assert got.shape == (274, 365, 3)
    assert np.array_equal(got, cv2.resize(img, None, fx=a, fy=a, interpolation=EXACT))


@pytest.mark.parametrize("sh,sw,dh,dw", [(1, 1, 1, 1), (5, 7, 1, 13), (17, 23, 7, 9), (16, 16, 33, 31)])
def test_resize_under_both_poisons(monkeypatch, sh, sw, dh, dw):
    src = np.random.default_rng(sh + dw).integers(0, 256, (3, sh, sw, 3), np.uint8)
    got = BC.under_both_poisons(monkeypatch, [_ops()], lambda fr, p, s: _ops().resize_linear_exact_u8(s, dh, dw),
                                lambda fr, p: (BC.framed_input(fr, p, src, name="src"),))[0]
    for k in range(3):
        assert np.array_equal(got[k], cv2.resize(src[k], (dw, dh), interpolation=EXACT)), k


# ---- the cases ---------------------------------------------------------------------------------------------------------------------
def case(name):
    """(frames, M, (Hc, Wc), megapix values): a 6-frame 1080 x 1920 sweep, a 3-frame 12 MP sweep and a ragged layout (frames
    of three sizes, rotated and in perspective)."""
    if name == "sweep1080":
        return GS.case("sweep1080") + ((0.1, 0.6),)
    if name == "sweep12mp":
        _, frames, _, H = SW.sweep(3, 3000, 4000, seed=6)
        return SL._chain(frames, H) + ((0.1, 0.6),)
    if name == "ragged":
        return SL.frame_case("warped") + ((0.004, 0.012),)
    raise KeyError(name)


_CACHE = {}


def scaled(name, q, finder):
    """(frames, M, canvas, a, the GPU's result) of case name at its q-th megapix value, cached across the tests."""
    key = (name, q, finder)
    if key not in _CACHE:
        frames, M, (Hc, Wc), mp = case(name)
        a = _mosaic().seam_scale([f.shape[:2] for f in frames], mp[q])
        assert a < 1
        _CACHE[key] = (frames, M, (Hc, Wc), a, _ops().mosaic_seam_masks(GS._cuda(frames), M, Hc, Wc, finder, scale=a))
    return _CACHE[key]


def _seam_inputs(frames, M, Hc, Wc, a):
    Ms, _, (Hs, Ws) = SS.seam_geometry(M, [f.shape[:2] for f in frames], Hc, Wc, a)
    return SM.fed([SS.resize_exact(f, fx=a) for f in frames], Ms, Hs, Ws), (Hs, Ws)


def _gpu_seams_by_frame(got):
    """The GPU's seam-scale seams as oracle/seam_scale.blend_masks takes them: (take_s, seams) of the frames fed at both
    scales (a frame fed only at seam scale does not reach the blend)."""
    take_s = [k for q, k in enumerate(got["take"]) if got["seam"][q].numel()]
    return take_s, [got["seam"][got["take"].index(k)].cpu().numpy() for k in take_s]


NAMES = ["sweep1080", "sweep12mp", "ragged"]


@pytest.mark.parametrize("finder", ["voronoi", "gc_color"])
@pytest.mark.parametrize("q", [0, 1])
@pytest.mark.parametrize("name", NAMES)
def test_seam_scale_seams_and_blend_masks(name, q, finder):
    frames, M, (Hc, Wc), a, got = scaled(name, q, finder)
    (take_s, imgs, masks, tls), canvas_s = _seam_inputs(frames, M, Hc, Wc, a)
    if finder == "voronoi":
        ref = SM.cv2_seams(masks, tls)
    else:
        ref, cuts = GC.restate(imgs, masks, tls)                 # T is canonical: the same for every maximum flow
        assert [int(c) for c in got["cut"]] == cuts
    for k, r in zip(take_s, ref):
        if k in got["take"]:
            assert np.array_equal(got["seam"][got["take"].index(k)].cpu().numpy(), r), ("seam", k)
    rois, _ = _mosaic().multiband_rois(M, [f.shape[:2] for f in frames], Hc, Wc)
    assert got["take"] == [k for k in range(len(frames)) if rois[k, 2] > rois[k, 0] and rois[k, 3] > rois[k, 1]]
    ts, ss = _gpu_seams_by_frame(got)
    want = SS.blend_masks(frames, M, Hc, Wc, a, ts, ss, got["seam_rois"], canvas_s)
    assert SL._equal([b.cpu().numpy() for b in got["blend"]], want)
    assert got["scale"] == a and any(((b > 0) & (b < 255)).any() for b in want)


def _by_frame(got, n):
    out = [None] * n
    for q, b in zip(got["take"], got["blend"]):
        out[q] = b
    return out


def _gain_maps(frames, seed):
    rng = np.random.default_rng(seed)
    return [rng.uniform(0.7, 1.3, (3, 4) if k % 2 else (2, 5, 3)).astype(np.float32) for k in range(len(frames))]


@pytest.mark.parametrize("comp", ["none", "gains", "maps"])
@pytest.mark.parametrize("name", ["sweep1080", "ragged"])
def test_blends_with_graded_masks_equal_the_oracle(name, comp):
    frames, M, (Hc, Wc), a, got = scaled(name, 0, "voronoi")
    bm_dev = _by_frame(got, len(frames))
    bm = [b.cpu().numpy() for b in got["blend"]]
    g = np.random.default_rng(9).uniform(0.6, 1.5, (len(frames), 3)) if comp == "gains" else None
    gm = _gain_maps(frames, 10) if comp == "maps" else None
    gm_dev = None if gm is None else [torch.from_numpy(m).cuda() for m in gm]
    out, mask = _ops().mosaic_multiband_u8(GS._cuda(frames), M, Hc, Wc, 5, gains=g, masks=bm_dev, gain_maps=gm_dev)
    ref, ref_mask = SS.multiband(frames, M, Hc, Wc, 5, bm, g, gm)
    assert np.array_equal(mask.cpu().numpy(), ref_mask) and np.array_equal(out.cpu().numpy(), ref)
    out, mask = _ops().mosaic_blend_u8(GS._cuda(frames), M, Hc, Wc, 64, gains=g, masks=bm_dev, gain_maps=gm_dev)
    ref, ref_mask = SS.feather(frames, M, Hc, Wc, 64, bm, g, gm)
    assert np.array_equal(mask.cpu().numpy(), ref_mask) and np.array_equal(out.cpu().numpy(), ref)


@pytest.mark.parametrize("finder", ["voronoi", "gc_color"])
def test_scale_one_is_the_full_resolution_call(finder):
    frames, M, (Hc, Wc) = SL.frame_case("sweep")
    a = _ops().mosaic_seam_masks(GS._cuda(frames), M, Hc, Wc, finder)
    b = _ops().mosaic_seam_masks(GS._cuda(frames), M, Hc, Wc, finder, scale=1.0)
    assert sorted(a) == sorted(b) and a["take"] == b["take"]
    assert all(np.array_equal(x.cpu().numpy(), y.cpu().numpy()) for x, y in zip(a["seam"] + a["blend"], b["seam"] + b["blend"]))


@pytest.mark.parametrize("finder", ["voronoi", "gc_color"])
def test_two_runs_are_bit_identical(finder):
    frames, M, (Hc, Wc), a, x = scaled("sweep1080", 0, finder)
    y = _ops().mosaic_seam_masks(GS._cuda(frames), M, Hc, Wc, finder, scale=a)
    assert all(np.array_equal(p.cpu().numpy(), q.cpu().numpy()) for p, q in zip(x["seam"] + x["blend"], y["seam"] + y["blend"]))


@pytest.mark.parametrize("finder", ["voronoi", "gc_color"])
def test_seam_scale_under_both_poisons(monkeypatch, finder):
    frames, M, (Hc, Wc) = SL.frame_case("warped")
    a = 0.43
    want = SS.masks(frames, M, Hc, Wc, a, finder)[1]

    def inputs(fr, p):
        return tuple(BC.framed_input(fr, p, f, name="frame%d" % k) for k, f in enumerate(frames))
    res = BC.under_both_poisons(monkeypatch, [_ops()], lambda fr, p, *f: _ops().mosaic_seam_masks(list(f), M, Hc, Wc, finder, scale=a),
                                inputs)[0]
    assert SL._equal(res["blend"], want)


# ---- build_mosaic and the CLI -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("finder", ["voronoi", "gc_color"])
@pytest.mark.parametrize("blend", ["feather", "multiband"])
def test_build_mosaic_with_seam_megapix(blend, finder):
    mosaic = _mosaic()
    _, frames, _, H = SW.sweep(3, 300, 400, seed=3)
    c = mosaic.build_mosaic(GS.TrueEstimator(H), GS._cuda(frames), blend=blend, seam=finder, seam_megapix=0.02)
    Hc, Wc = c["mask"].shape
    a = c["seam_scale"]
    assert a == mosaic.seam_scale([(300, 400)], 0.02) < 1 and c["last_ms"]["seam"] > 0
    take, bm, _ = SS.masks(frames, c["M"], Hc, Wc, a, finder)
    ref = SS.multiband(frames, c["M"], Hc, Wc, 5, bm)[0] if blend == "multiband" else SS.feather(frames, c["M"], Hc, Wc, 64, bm)[0]
    assert np.array_equal(c["mosaic"].cpu().numpy(), ref)
    full = mosaic.build_mosaic(GS.TrueEstimator(H), GS._cuda(frames), blend=blend, seam=finder, seam_megapix=1.0)
    plain = mosaic.build_mosaic(GS.TrueEstimator(H), GS._cuda(frames), blend=blend, seam=finder)
    assert full["seam_scale"] == 1.0 and np.array_equal(full["mosaic"].cpu().numpy(), plain["mosaic"].cpu().numpy())


def test_cli_end_to_end(tmp_path):
    import mosaic_images as cli
    raw = tmp_path / "raw"
    raw.mkdir()
    _, frames, _, _ = SW.sweep(3, 240, 320, seed=9)
    names = ["DSC_%04d.JPG" % k for k in range(3)]
    for nm, f in zip(names, frames):
        cv2.imwrite(str(raw / nm), f[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, 95])
    out = tmp_path / "mosaic"
    assert cli.main(["--frames", str(raw), "--out_dir", str(out), "--seeded_weights", "True", "--model_dir", str(tmp_path / "none"),
                     "--blend", "multiband", "--seam", "gc_color", "--seam_megapix", "0.02"]) == 0
    head = (out / "mosaic.txt").read_text().splitlines()[0].split()
    a = float(head[-1])
    assert head[5:-1] == ["blend", "multiband", "5", "seam", "gc_color"] and a == _mosaic().seam_scale([(240, 320)], 0.02)
    Hc, Wc = int(head[1]), int(head[2])
    imgs, Ms = [], []
    for ln, nm in zip((out / "mosaic.txt").read_text().splitlines()[1:], names):
        parts = ln.split()
        if parts[1] == "kept":
            imgs.append(cv2.imread(str(raw / nm))[..., ::-1].copy())
            Ms.append(np.array([float(v) for v in parts[2:11]]).astype(np.float32).astype(np.float64).reshape(3, 3))
    _, bm, _ = SS.masks(imgs, np.stack(Ms), Hc, Wc, a, "gc_color")
    mos, _ = SS.multiband(imgs, np.stack(Ms), Hc, Wc, 5, bm)
    assert (out / "mosaic.jpg").read_bytes() == _ops().encode_jpeg(np.ascontiguousarray(mos[..., ::-1])[None])[0]


# ---- the numbers the feature reports ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,h,w,seed,megapix", [(5, 1080, 1920, 3, 0.1), (6, 480, 640, 0, 0.1), (6, 480, 640, 0, 0.03)])
def test_pixels_left_without_weight(n, h, w, seed, megapix):
    """Valid full-resolution pixels that no frame's graded mask covers (the seam-scale frames end up to 1 / (2a) px short of
    the full ones): reported, and all of them near the union's outside."""
    _, frames, _, H = SW.sweep(n, h, w, seed=seed)
    frames, M, (Hc, Wc) = SL._chain(frames, H)
    a = _mosaic().seam_scale([(h, w)], megapix)
    got = _ops().mosaic_seam_masks(GS._cuda(frames), M, Hc, Wc, "voronoi", scale=a)
    valid = np.zeros((Hc, Wc), bool)
    on = np.zeros((Hc, Wc), bool)
    for b, k in zip(got["blend"], got["take"]):
        x0, y0, x1, y1 = (int(v) for v in got["rois"][k])
        roi_valid, _ = SM.OM.validity_weight(_mosaic().multiband_rois(M, [f.shape[:2] for f in frames], Hc, Wc)[1][k], h, w, y1 - y0, x1 - x0, 0)
        valid[y0:y1, x0:x1] |= roi_valid
        on[y0:y1, x0:x1] |= b.cpu().numpy() != 0
    lost = valid & ~on
    outside = cv2.distanceTransform(np.where(valid, 255, 0).astype(np.uint8), cv2.DIST_L2, 3)
    far = float(outside[lost].max()) if lost.any() else 0.0
    print("no weight: %d x %dx%d at %.3g MP (a = %.4f): %d of %d valid pixels, farthest %.1f px from the union's outside"
          % (n, h, w, megapix, a, int(lost.sum()), int(valid.sum()), far))
    assert far <= 2.0 / a + 2


def test_drifting_sweep_score_at_a_tenth_of_a_megapixel():
    """test_gpu_seam_gc's drifting sweep with the seams found at 0.1 MP: the mean absolute difference to the true texture
    over the overlaps, both finders and both blends, beside the full-resolution finders."""
    mosaic = _mosaic()
    tex, frames, A, H = SW.sweep(6, 480, 640, seed=11)
    rng = np.random.default_rng(11)
    Hp = np.stack([T(*rng.uniform(-3, 3, 2)) @ h for h in H])
    G, r = mosaic.chain_to_reference(Hp)
    M, (Hc, Wc), kept = mosaic.canvas([f.shape[:2] for f in frames], G, r)
    _, _, masks, tls = SM.fed(frames, M, Hc, Wc)
    seen = cv2.warpPerspective(tex, A[r] @ np.linalg.inv(M[r]), (Wc, Hc), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP)
    cover = np.zeros((Hc, Wc), np.int32)
    for m, (x, y) in zip(masks, tls):
        cover[y:y + m.shape[0], x:x + m.shape[1]] += m != 0
    over = cover >= 2
    res = {}
    for scale in (1.0, mosaic.seam_scale([(480, 640)], 0.1)):
        for finder in ("voronoi", "gc_color"):
            bm = _by_frame(_ops().mosaic_seam_masks(GS._cuda(frames), M, Hc, Wc, finder, scale=scale), len(frames))
            for blend in ("multiband", "feather"):
                if blend == "multiband":
                    out, _ = _ops().mosaic_multiband_u8(GS._cuda(frames), M, Hc, Wc, 5, masks=bm)
                else:
                    out, _ = _ops().mosaic_blend_u8(GS._cuda(frames), M, Hc, Wc, 64, masks=bm)
                res[(scale, finder, blend)] = float(np.abs(out.cpu().numpy().astype(np.int32) - seen.astype(np.int32))[over].mean())
    print("drifting sweep, overlap MAD to the texture: " + ", ".join("a=%.4f %s %s %.3f" % (k + (v,)) for k, v in res.items()))
    assert all(np.isfinite(v) for v in res.values())
