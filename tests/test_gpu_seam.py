"""GPU tests of the mosaic's seams: udh_mosaic_seam_masks_u8's seam and blend masks against cv2.detail's Voronoi seam
finder byte for byte (hand-built pairs, warped and clipped frames, 190 pairs, a 1080 x 1920 sweep, a pair of 12 MP frames
with distances past 4000 px), both blends with seams against their oracles (oracle/seam.py), seam="none" against the
un-seamed bytes, run independence, mosaic_images.py --seam end to end, and one quality number."""
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
import test_seam_logic as SL  # noqa: E402
from oracle import exposure as EX  # noqa: E402
from oracle import multiband as MB  # noqa: E402
from oracle import seam as SM  # noqa: E402

pytestmark = pytest.mark.gpu
T = SL.T


def _cuda(frames):
    return [torch.from_numpy(np.ascontiguousarray(f)).cuda() for f in frames]


def case(name):
    """(frames uint8 RGB, M, (Hc, Wc)): test_seam_logic's frame cases, frames placed as its hand-built mask cases, a
    1080 x 1920 sweep and a pair of 12 MP frames."""
    rng = np.random.default_rng(sum(map(ord, name)))
    if name in SL.FRAME_CASES:
        return SL.frame_case(name)
    if name == "tie":                                          # a 7-px overlap (with the ROIs' margins, 10 px)
        sizes, M, canvas = [(20, 30), (20, 30)], [T(1, 1), T(24, 1)], (22, 56)
    elif name == "order":
        sizes, M, canvas = [(30, 40)] * 3, [T(1, 1), T(26, 7), T(11, 23)], (56, 68)
    elif name == "contained":                                  # frame 1 inside frame 0, frame 2 inside frame 1
        sizes, M, canvas = [(40, 50), (20, 24), (6, 6)], [T(1, 1), T(13, 10), T(21, 16)], (42, 52)
    elif name == "no_unique":                                  # the same frame twice
        sizes, M, canvas = [(12, 15), (12, 15)], [T(3, 4), T(3, 4)], (18, 20)
    elif name == "sweep1080":
        _, frames, _, H = SW.sweep(6, 1080, 1920, seed=4)
        return SL._chain(frames, H)
    elif name == "pair12mp":                                   # 1000 x 12000 frames one pixel apart: the seam lies ~6000 px
        tex = SW.texture(rng, 1002, 12004)                     # from both frames' own pixels
        return [tex[1:1001, 1:12001].copy(), tex[1:1001, 2:12002].copy()], np.stack([T(0, 0), T(1, 0)]), (1000, 12001)
    else:
        raise KeyError(name)
    frames = [rng.integers(0, 256, (h, w, 3), np.uint8) for h, w in sizes]
    return frames, np.stack(M), canvas


CASES = ["tie", "order", "contained", "no_unique"] + SL.FRAME_CASES
BIG = ["sweep1080", "pair12mp"]


# ---- seam and blend masks ------------------------------------------------------------------------------------------------
def _check_masks(frames, M, Hc, Wc):
    from unsuperviseddeephomographyral2018_b200 import ops
    got = ops.mosaic_seam_masks(_cuda(frames), M, Hc, Wc)
    take, _, masks, tls = SM.fed(frames, M, Hc, Wc)
    assert got["take"] == take
    seams = SM.cv2_seams(masks, tls)
    for k, (s, b, ref_s, ref_b) in enumerate(zip(got["seam"], got["blend"], seams, SM.blend_masks(seams, masks))):
        assert np.array_equal(s.cpu().numpy(), ref_s), ("seam", k)
        assert np.array_equal(b.cpu().numpy(), ref_b), ("blend", k)
    return got, masks, seams


@pytest.mark.parametrize("name", CASES + BIG)
def test_seam_and_blend_masks_equal_cv2(name):
    frames, M, (Hc, Wc) = case(name)
    got, masks, seams = _check_masks(frames, M, Hc, Wc)
    if name == "contained":
        assert not seams[1].any() and not seams[2].any()
    if name == "no_unique":
        assert not seams[0].any() and np.array_equal(seams[1], masks[1])
    if name == "stacked":
        assert len(SM.pairs([(int(r[0]), int(r[1])) for r in got["rois"]], [m.shape for m in masks])) == 190
    if name == "pair12mp":                                     # frame 0 keeps the left half: distances past 4000 px decide it
        keep = np.flatnonzero(seams[0][500])
        assert keep.max() > 5500 and seams[0][500, 5000:keep.max()].all()


def test_distance_cap_would_change_the_12mp_pair():
    """On the 12 MP pair the exact rule and a 4095-capped one disagree, so the check above sees distances past 4000."""
    frames, M, (Hc, Wc) = case("pair12mp")
    _, _, masks, tls = SM.fed(frames, M, Hc, Wc)
    exact = SM.restate(masks, tls)
    l1 = SM.l1_distance
    try:
        SM.l1_distance = lambda src: np.minimum(l1(src), 4095)
        capped = SM.restate(masks, tls)
    finally:
        SM.l1_distance = l1
    assert not np.array_equal(exact[0], capped[0])


def test_two_runs_are_bit_identical():
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case("stacked")
    a = ops.mosaic_seam_masks(_cuda(frames), M, Hc, Wc)
    b = ops.mosaic_seam_masks(_cuda(frames), M, Hc, Wc)
    assert all(np.array_equal(x.cpu().numpy(), y.cpu().numpy()) for x, y in zip(a["seam"] + a["blend"], b["seam"] + b["blend"]))


# ---- the blends with seams -----------------------------------------------------------------------------------------------
def _blend_masks(frames, M, Hc, Wc):
    """Blend masks [n] aligned with the frames (None where not fed), from 3-channel copies of the frames."""
    from unsuperviseddeephomographyral2018_b200 import ops
    rgb = [f if f.ndim == 3 and f.shape[2] == 3 else np.repeat(f.reshape(f.shape[0], f.shape[1], 1), 3, 2) for f in frames]
    s = ops.mosaic_seam_masks(_cuda(rgb), M, Hc, Wc)
    out = [None] * len(frames)
    for q, b in zip(s["take"], s["blend"]):
        out[q] = b
    return out


@pytest.mark.parametrize("gains", [False, True])
@pytest.mark.parametrize("name", ["order", "warped", "stacked", "sweep"])
def test_multiband_with_seams_equals_the_oracle(name, gains):
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case(name)
    g = np.random.default_rng(7).uniform(0.6, 1.5, (len(frames), 3)) if gains else None
    out, mask = ops.mosaic_multiband_u8(_cuda(frames), M, Hc, Wc, 5, gains=g, masks=_blend_masks(frames, M, Hc, Wc))
    ref, ref_mask = SM.multiband(frames, M, Hc, Wc, 5, g)
    assert np.array_equal(mask.cpu().numpy(), ref_mask) and np.array_equal(out.cpu().numpy(), ref)


@pytest.mark.parametrize("gains", [False, True])
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("name", ["clipped", "warped", "stacked", "sweep"])
def test_feathered_blend_with_seams_equals_the_oracle(name, C, gains):
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case(name)
    frames = [f[..., :C].copy() for f in frames]
    g = np.random.default_rng(8).uniform(0.6, 1.5, (len(frames), 3)) if gains else None
    out, mask = ops.mosaic_blend_u8(_cuda(frames), M, Hc, Wc, 64, gains=g, masks=_blend_masks(frames, M, Hc, Wc))
    ref, ref_mask = SM.feather(frames, M, Hc, Wc, 64, g)
    assert np.array_equal(mask.cpu().numpy(), ref_mask) and np.array_equal(out.cpu().numpy(), ref)


# ---- build_mosaic ----------------------------------------------------------------------------------------------------------
class TrueEstimator(object):
    """est.estimate returning given pair homographies (the chain the mosaic is built from)."""

    def __init__(self, H):
        self.H, self.last_ms = H, dict(prep=0.0, forward=0.0)

    def estimate(self, a, b):
        return self.H, None, None


@pytest.mark.parametrize("blend", ["feather", "multiband"])
def test_seam_none_gives_the_unseamed_bytes(blend):
    from unsuperviseddeephomographyral2018_b200 import mosaic
    _, frames, _, H = SW.sweep(4, 120, 160, seed=3)
    est = TrueEstimator(H)
    a = mosaic.build_mosaic(est, _cuda(frames), blend=blend)
    b = mosaic.build_mosaic(est, _cuda(frames), blend=blend, seam="none")
    c = mosaic.build_mosaic(est, _cuda(frames), blend=blend, seam="voronoi")
    assert "seam" not in a["last_ms"] and "seam" not in b["last_ms"] and c["last_ms"]["seam"] > 0
    assert np.array_equal(a["mosaic"].cpu().numpy(), b["mosaic"].cpu().numpy())
    Hc, Wc = a["mask"].shape
    ref = MB.blend(frames, a["M"], Hc, Wc, 5)[0] if blend == "multiband" else SL_feather(frames, a["M"], Hc, Wc)
    assert np.array_equal(a["mosaic"].cpu().numpy(), ref)
    seamed = SM.multiband(frames, c["M"], Hc, Wc, 5)[0] if blend == "multiband" else SM.feather(frames, c["M"], Hc, Wc, 64)[0]
    assert np.array_equal(c["mosaic"].cpu().numpy(), seamed)
    assert not np.array_equal(a["mosaic"].cpu().numpy(), seamed)
    with pytest.raises(ValueError, match="seam"):
        mosaic.build_mosaic(est, _cuda(frames), seam="dp")


def SL_feather(frames, M, Hc, Wc):
    from oracle import mosaic as OM
    return OM.blend(frames, M, Hc, Wc, 64)[0]


# ---- the CLI -------------------------------------------------------------------------------------------------------------------
def test_cli_end_to_end(tmp_path):
    import mosaic_images as cli
    from unsuperviseddeephomographyral2018_b200 import ops
    raw = tmp_path / "raw"
    raw.mkdir()
    _, frames, _, _ = SW.sweep(4, 240, 320, seed=9)
    frames = [EX.apply(f, e) for f, e in zip(frames, (0.6, 0.7, 0.85, 0.65))]
    names = ["DSC_%04d.JPG" % k for k in range(4)]
    for nm, f in zip(names, frames):
        cv2.imwrite(str(raw / nm), f[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, 95])
    out = tmp_path / "mosaic"
    assert cli.main(["--frames", str(raw), "--out_dir", str(out), "--seeded_weights", "True", "--model_dir", str(tmp_path / "none"),
                     "--blend", "multiband", "--compensate", "channels", "--seam", "voronoi"]) == 0
    txt = (out / "mosaic.txt").read_text().splitlines()
    head = txt[0].split()
    assert head[5:] == ["blend", "multiband", "5", "compensate", "channels", "1", "seam", "voronoi"]
    Hc, Wc = int(head[1]), int(head[2])
    imgs, Ms, gains = [], [], []
    for ln, nm in zip(txt[1:], names):
        parts = ln.split()
        if parts[1] == "kept":
            imgs.append(cv2.imread(str(raw / nm))[..., ::-1].copy())
            Ms.append(np.array([float(v) for v in parts[2:11]]).astype(np.float32).astype(np.float64).reshape(3, 3))
            gains.append([float(v) for v in parts[11:]])
    M = np.stack(Ms)
    assert np.array_equal(np.array(gains), EX.gains(imgs, M, Hc, Wc, "channels", 1))   # from the un-seamed masks
    mos, _ = SM.multiband(imgs, M, Hc, Wc, 5, np.array(gains))
    assert (out / "mosaic.jpg").read_bytes() == ops.encode_jpeg(np.ascontiguousarray(mos[..., ::-1])[None])[0]


# ---- one quality number --------------------------------------------------------------------------------------------------------
def test_seams_on_a_drifting_sweep_quality():
    """A textured sweep whose chain is perturbed by a few pixels per pair: the mean absolute difference to the true
    texture (as the reference frame sees it) over the pixels two or more frames cover, multi-band with and without seams.
    Reported either way; the test checks only that it is computed."""
    from unsuperviseddeephomographyral2018_b200 import mosaic, ops
    tex, frames, A, H = SW.sweep(6, 480, 640, seed=11)
    rng = np.random.default_rng(11)
    Hp = np.stack([T(*rng.uniform(-3, 3, 2)) @ h for h in H])
    G, r = mosaic.chain_to_reference(Hp)
    M, (Hc, Wc), kept = mosaic.canvas([f.shape[:2] for f in frames], G, r)
    seen = cv2.warpPerspective(tex, A[r] @ np.linalg.inv(M[r]), (Wc, Hc), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP)
    take, _, masks, tls = SM.fed(frames, M, Hc, Wc)
    cover = np.zeros((Hc, Wc), np.int32)
    for m, (x, y) in zip(masks, tls):
        cover[y:y + m.shape[0], x:x + m.shape[1]] += m != 0
    over = cover >= 2
    res = {}
    for label, masks_arg in (("without seams", None), ("with seams", _blend_masks(frames, M, Hc, Wc))):
        out, _ = ops.mosaic_multiband_u8(_cuda(frames), M, Hc, Wc, 5, masks=masks_arg)
        res[label] = float(np.abs(out.cpu().numpy().astype(np.int32) - seen.astype(np.int32))[over].mean())
    print("drifting sweep, overlap MAD to the texture: %.3f without seams, %.3f with seams (%.1f %% of the canvas in overlaps)"
          % (res["without seams"], res["with seams"], 100 * over.mean()))
    assert over.any() and all(np.isfinite(v) for v in res.values())
