"""GPU tests of the mosaic's block exposure compensation: udh_mosaic_exposure_block_stats_u8 against the restated block
statistics exactly, the conjugate-gradient gains and the filtered maps against cv2.detail's block compensators, both
blends with gain maps (with and without seams, both modes) against oracle/exposure_blocks.py byte for byte, unit maps,
run independence, the solver on a 1080 x 1920 sweep, mosaic_images.py --compensate gain_blocks end to end, and one
quality number."""
import os
import sys

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _mosaic_sweep as SW  # noqa: E402
import test_exposure_blocks_logic as XL  # noqa: E402
import test_seam_logic as SL  # noqa: E402
from oracle import exposure as EX  # noqa: E402
from oracle import exposure_blocks as XB  # noqa: E402
from oracle import seam as SM  # noqa: E402

pytestmark = pytest.mark.gpu


def _cuda(frames):
    return [torch.from_numpy(np.ascontiguousarray(f)).cuda() for f in frames]


def case(name):
    """(frames uint8 RGB with vignetting and exposure steps, M, (Hc, Wc))."""
    if name == "sweep1080":
        _, frames, _, H = SW.sweep(4, 1080, 1920, seed=4)
        frames, M, canvas = SL._chain(frames, H)
    else:
        frames, M, canvas = SL.frame_case(name)
    gains = [1.0, 0.75, 1.2, 0.9, 1.1, 0.8]
    return [XL.vignette(f.astype(np.float64), 0.3, gains[k % 6]) for k, f in enumerate(frames)], M, canvas


CASES = ["clipped", "warped", "stacked", "sweep"]


# ---- statistics -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("feeds", [0, 2])
@pytest.mark.parametrize("block", [16, 32, 48])
@pytest.mark.parametrize("name", CASES)
def test_block_statistics_equal_the_restatement(name, block, feeds):
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case(name)
    take, imgs, masks, tls = EX.fed(frames, M, Hc, Wc)
    bi, bm, bt, grids = XB.blocks(imgs, masks, tls, block, block)
    hist = np.random.default_rng(block).uniform(0.7, 1.4, (feeds, len(bi), 3)) if feeds else None
    cur = [np.asarray(i) for i in bi]
    for t in range(feeds):
        cur = [EX.apply(img, g) for img, g in zip(cur, hist[t])]
    ref = {(p["i"], p["j"]): p for p in EX.pair_stats(cur, bm, bt, "exact")}
    got = ops.mosaic_exposure_block_stats(_cuda(frames), M, Hc, Wc, block, history=hist)
    assert sorted(zip(got["a"].tolist(), got["b"].tolist())) == sorted(ref)
    for q, (a, b) in enumerate(zip(got["a"].tolist(), got["b"].tolist())):
        p = ref[(a, b)]
        assert got["count"][q] == p["count"], (a, b)
        assert np.array_equal(got["sums"][q], p["sums"]), (a, b)
        assert np.array_equal(got["norms"][q], p["norms"]), (a, b)


# ---- gains and maps ----------------------------------------------------------------------------------------------------------
def _midpoint_margin(g):
    """Distance of each float64 gain from the nearest float32 rounding midpoint."""
    f = g.astype(np.float32).astype(np.float64)
    up = np.nextafter(g.astype(np.float32), np.float32(np.inf)).astype(np.float64)
    dn = np.nextafter(g.astype(np.float32), np.float32(-np.inf)).astype(np.float64)
    return np.minimum(np.abs(g - (f + up) / 2), np.abs(g - (f + dn) / 2))


@pytest.mark.parametrize("feeds", [1, 3])
@pytest.mark.parametrize("block", [16, 32, 48])
@pytest.mark.parametrize("mode", ["gain", "channels"])
@pytest.mark.parametrize("name", CASES)
def test_gains_and_maps_equal_cv2(name, mode, block, feeds):
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case(name)
    take, imgs, masks, tls = EX.fed(frames, M, Hc, Wc)
    ref_maps, _ = XB.cv2_maps(imgs, masks, tls, mode, feeds, block)
    _, g_cv2, _, _ = XB.restate(imgs, masks, tls, mode, feeds, block)       # cv2's gains bit for bit (test_exposure_blocks_logic)
    got = ops.mosaic_exposure_block_gains(_cuda(frames), M, Hc, Wc, mode, feeds, block)
    assert got["take"] == take
    err = np.abs(got["gains"] - g_cv2).max()
    assert err <= 1e-12, err
    assert all(r <= ops.EXPOSURE_BLOCK_TOL for r in got["residual"])
    margin = _midpoint_margin(g_cv2)
    if (margin > 1e-12).all():
        for k, r in zip(take, ref_maps):
            assert XL._bits_equal(got["maps"][k].cpu().numpy(), r)
    else:                                                    # a gain within the solver's error of a float32 tie
        assert (got["gains"].astype(np.float32) == g_cv2.astype(np.float32))[margin > 1e-12].all()


def test_frames_without_overlap_get_unit_maps():
    from unsuperviseddeephomographyral2018_b200 import ops
    rng = np.random.default_rng(0)
    frames = [rng.integers(0, 256, (40, 50, 3), np.uint8) for _ in range(2)]
    M = np.stack([SL.T(1, 1), SL.T(80, 1)])
    maps = ops.mosaic_exposure_gain_maps(_cuda(frames), M, 45, 140, "channels", 2, 16)
    assert all((m.cpu().numpy() == 1).all() for m in maps)


def test_two_runs_are_bit_identical():
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case("stacked")
    a = ops.mosaic_exposure_block_gains(_cuda(frames), M, Hc, Wc, "gain", 2, 16)
    b = ops.mosaic_exposure_block_gains(_cuda(frames), M, Hc, Wc, "gain", 2, 16)
    assert np.array_equal(a["gains"].view(np.uint64), b["gains"].view(np.uint64)) and a["iters"] == b["iters"]
    assert all(np.array_equal(x.cpu().numpy(), y.cpu().numpy()) for x, y in zip(a["maps"], b["maps"]))


def test_solver_converges_on_a_1080p_sweep():
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case("sweep1080")
    st = ops.mosaic_exposure_block_stats(_cuda(frames), M, Hc, Wc, 32)
    sa, sb = st["norms"][:, 0], st["norms"][:, 1]
    nblocks = int(st["boff"][-1] + st["blocks"][-1, 2] * st["blocks"][-1, 3])
    keep, ptr, col, val, rhs = ops.exposure_block_system(nblocks, st["a"], st["b"], st["count"], sa, sb)
    x, it, res = ops.exposure_block_solve(ptr, col, val, rhs, torch.device("cuda"))
    print("1080 x 1920 sweep, 32 px blocks: %d blocks, %d unknowns, %d nonzeros, %d iterations, |r| / |b| = %.2e"
          % (nblocks, len(keep), len(val), it, res))
    assert len(keep) > 1000 and res <= ops.EXPOSURE_BLOCK_TOL and it < ops.EXPOSURE_BLOCK_MAX_ITER
    sp = pytest.importorskip("scipy.sparse")
    spl = pytest.importorskip("scipy.sparse.linalg")
    ref = spl.spsolve(sp.csr_matrix((val, col, ptr), shape=(len(keep), len(keep))).tocsc(), rhs)
    assert np.abs(x - ref).max() <= 1e-12


# ---- the blends -------------------------------------------------------------------------------------------------------------------
def _blend_masks(frames, M, Hc, Wc):
    from unsuperviseddeephomographyral2018_b200 import ops
    s = ops.mosaic_seam_masks(_cuda(frames), M, Hc, Wc)
    out = [None] * len(frames)
    for q, b in zip(s["take"], s["blend"]):
        out[q] = b
    return out


@pytest.mark.parametrize("seam", [False, True])
@pytest.mark.parametrize("mode", ["gain", "channels"])
@pytest.mark.parametrize("name", CASES)
def test_multiband_with_gain_maps_equals_the_oracle(name, mode, seam):
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case(name)
    maps = ops.mosaic_exposure_gain_maps(_cuda(frames), M, Hc, Wc, mode, 2, 16)
    ref_maps = XB.maps(frames, M, Hc, Wc, mode, 2, 16)
    bm = _blend_masks(frames, M, Hc, Wc) if seam else None
    out, mask = ops.mosaic_multiband_u8(_cuda(frames), M, Hc, Wc, 5, masks=bm, gain_maps=maps)
    host = [None if m is None else m.cpu().numpy() for m in maps]
    take = [k for k in range(len(frames)) if host[k] is not None]
    ref, ref_mask = XB.multiband(frames, M, Hc, Wc, 5, host, None if bm is None else [bm[k].cpu().numpy() for k in take])
    assert np.array_equal(mask.cpu().numpy(), ref_mask) and np.array_equal(out.cpu().numpy(), ref)
    same = all(XL._bits_equal(a, b) for a, b in zip([host[k] for k in take], [ref_maps[k] for k in take]))
    print("%s %s: GPU maps %s the restated maps" % (name, mode, "equal" if same else "differ from"))


@pytest.mark.parametrize("seam", [False, True])
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("mode", ["gain", "channels"])
@pytest.mark.parametrize("name", CASES)
def test_feathered_blend_with_gain_maps_equals_the_oracle(name, mode, C, seam):
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case(name)
    maps = ops.mosaic_exposure_gain_maps(_cuda(frames), M, Hc, Wc, mode, 1, 32)
    bm = _blend_masks(frames, M, Hc, Wc) if seam else None
    fr = [f[..., :C].copy() for f in frames]
    out, mask = ops.mosaic_blend_u8(_cuda(fr), M, Hc, Wc, 64, masks=bm, gain_maps=maps)
    host = [None if m is None else m.cpu().numpy() for m in maps]
    take = [k for k in range(len(frames)) if host[k] is not None]
    ref, ref_mask = XB.feather(fr, M, Hc, Wc, 64, host, None if bm is None else [bm[k].cpu().numpy() for k in take])
    assert np.array_equal(mask.cpu().numpy(), ref_mask) and np.array_equal(out.cpu().numpy(), ref)


@pytest.mark.parametrize("blend", ["feather", "multiband"])
def test_unit_maps_give_the_uncompensated_bytes(blend):
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case("warped")
    maps = [None if m is None else torch.ones_like(m) for m in ops.mosaic_exposure_gain_maps(_cuda(frames), M, Hc, Wc, "channels", 1, 32)]
    if blend == "feather":
        a = ops.mosaic_blend_u8(_cuda(frames), M, Hc, Wc, 64, gain_maps=maps)
        b = ops.mosaic_blend_u8(_cuda(frames), M, Hc, Wc, 64)
    else:
        a = ops.mosaic_multiband_u8(_cuda(frames), M, Hc, Wc, 5, gain_maps=maps)
        b = ops.mosaic_multiband_u8(_cuda(frames), M, Hc, Wc, 5)
    assert all(np.array_equal(x.cpu().numpy(), y.cpu().numpy()) for x, y in zip(a, b))


# ---- build_mosaic and the CLI -------------------------------------------------------------------------------------------------
class TrueEstimator(object):
    def __init__(self, H):
        self.H, self.last_ms = H, dict(prep=0.0, forward=0.0)

    def estimate(self, a, b):
        return self.H, None, None


def test_cli_end_to_end(tmp_path):
    import mosaic_images as cli
    from unsuperviseddeephomographyral2018_b200 import ops
    raw = tmp_path / "raw"
    raw.mkdir()
    _, frames, _, _ = SW.sweep(4, 240, 320, seed=9)
    frames = [XL.vignette(f.astype(np.float64), 0.3, e) for f, e in zip(frames, (0.6, 0.7, 0.85, 0.65))]
    names = ["DSC_%04d.JPG" % k for k in range(4)]
    for nm, f in zip(names, frames):
        cv2.imwrite(str(raw / nm), f[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, 95])
    out = tmp_path / "mosaic"
    assert cli.main(["--frames", str(raw), "--out_dir", str(out), "--seeded_weights", "True", "--model_dir", str(tmp_path / "none"),
                     "--blend", "multiband", "--compensate", "gain_blocks", "--compensate_feeds", "2", "--compensate_block", "48",
                     "--seam", "voronoi"]) == 0
    txt = (out / "mosaic.txt").read_text().splitlines()
    head = txt[0].split()
    assert head[5:] == ["blend", "multiband", "5", "compensate", "gain_blocks", "2", "48", "seam", "voronoi"]
    Hc, Wc = int(head[1]), int(head[2])
    imgs, Ms = [], []
    for ln, nm in zip(txt[1:], names):
        parts = ln.split()
        assert len(parts) == 11
        if parts[1] == "kept":
            imgs.append(cv2.imread(str(raw / nm))[..., ::-1].copy())
            Ms.append(np.array([float(v) for v in parts[2:11]]).astype(np.float32).astype(np.float64).reshape(3, 3))
    assert len(imgs) == 4
    M = np.stack(Ms)
    saved = np.load(out / "gain_maps.npz")
    maps = [saved[nm] for nm in names]
    take, fimgs, fmasks, tls = EX.fed(imgs, M, Hc, Wc)
    bm = SM.blend_masks(SM.cv2_seams(fmasks, tls), fmasks)
    mos, _ = XB.multiband(imgs, M, Hc, Wc, 5, maps, bm)
    assert (out / "mosaic.jpg").read_bytes() == ops.encode_jpeg(np.ascontiguousarray(mos[..., ::-1])[None])[0]


def test_build_mosaic_block_modes():
    from unsuperviseddeephomographyral2018_b200 import mosaic
    _, frames, _, H = SW.sweep(4, 120, 160, seed=3)
    est = TrueEstimator(H)
    a = mosaic.build_mosaic(est, _cuda(frames), compensate="channels_blocks", compensate_block=16)
    assert (a["gains"] == 1).all() and len(a["gain_maps"]) == 4 and a["last_ms"]["compensate"] > 0
    b = mosaic.build_mosaic(est, _cuda(frames))
    assert "gain_maps" not in b
    with pytest.raises(ValueError, match="compensate"):
        mosaic.build_mosaic(est, _cuda(frames), compensate="blocks")


# ---- one quality number --------------------------------------------------------------------------------------------------------
def test_vignetted_sweep_quality():
    """A sweep with 30 % radial vignetting and exposure steps: the mean absolute difference between overlapping ROI warps
    after compensation (none, gain, gain_blocks; 2 feeds, 32 px blocks).  Reported; the test checks only that block
    gains reduce it."""
    from unsuperviseddeephomographyral2018_b200 import ops
    _, frames, _, H = SW.sweep(5, 480, 640, seed=12)
    frames, M, (Hc, Wc) = SL._chain(frames, H)
    frames = [XL.vignette(f.astype(np.float64), 0.3, e) for f, e in zip(frames, (1.0, 0.8, 1.15, 0.9, 1.05))]
    take, imgs, masks, tls = EX.fed(frames, M, Hc, Wc)

    def mad(imgs):
        tot, n = 0.0, 0
        for i, j, (x0, y0, x1, y1) in EX.pairs([(x, y, x + m.shape[1], y + m.shape[0]) for (x, y), m in zip(tls, masks)]):
            if i == j:
                continue
            si = (slice(y0 - tls[i][1], y1 - tls[i][1]), slice(x0 - tls[i][0], x1 - tls[i][0]))
            sj = (slice(y0 - tls[j][1], y1 - tls[j][1]), slice(x0 - tls[j][0], x1 - tls[j][0]))
            both = (masks[i][si] != 0) & (masks[j][sj] != 0)
            tot += np.abs(imgs[i][si].astype(np.int32) - imgs[j][sj].astype(np.int32))[both].sum()
            n += both.sum() * 3
        return tot / n

    g = ops.mosaic_exposure_gains(_cuda(frames), M, Hc, Wc, "gain", 2)
    maps = ops.mosaic_exposure_gain_maps(_cuda(frames), M, Hc, Wc, "gain", 2, 32)
    res = dict(none=mad(imgs), gain=mad([EX.apply(i, g[k]) for i, k in zip(imgs, take)]),
               gain_blocks=mad([XB.apply_map(i, maps[k].cpu().numpy()) for i, k in zip(imgs, take)]))
    print("vignetted sweep, overlap MAD: none %.2f, gain %.2f, gain_blocks %.2f" % (res["none"], res["gain"], res["gain_blocks"]))
    assert res["gain_blocks"] < res["none"]
