"""Host-side tests of the graph-cut seams: the NumPy restatement (oracle/seam_gc.py) against cv2.detail's
GraphCutSeamFinder(COST_COLOR) byte for byte where every pair's minimum cut is unique, cv2 inside the restatement's
lattice bounds where it is not, the visiting order, contained frames, pairs without source or sink pixels, the
certificate checker, and mosaic_images.py's --seam gc_color and mosaic.txt."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _mosaic_sweep as SW  # noqa: E402
import test_seam_logic as SL  # noqa: E402

cv2 = pytest.importorskip("cv2")
from oracle import seam as SM  # noqa: E402
from oracle import seam_gc as GC  # noqa: E402

T = SL.T


def gc_case(name):
    """(frames uint8 RGB, M [n,3,3], (Hc, Wc)) of a named graph-cut case."""
    rng = np.random.default_rng(sum(map(ord, name)) + 1)
    if name in ("clipped", "warped"):
        return SL.frame_case(name)
    if name == "noisy":                                        # a textured pair, independent noise in each frame
        tex = SW.texture(rng, 90, 140)
        a, b = tex[:80, :90], tex[5:85, 40:130]
        frames = [np.clip(f.astype(np.int32) + rng.integers(-20, 21, f.shape), 0, 255).astype(np.uint8) for f in (a, b)]
        return frames, np.stack([T(1, 1), T(41, 6)]), (92, 136)
    if name == "order":                                        # three noise frames, each overlapping both others
        frames = [rng.integers(0, 256, (30, 40, 3), np.uint8) for _ in range(3)]
        return frames, np.stack([T(1, 1), T(26, 7), T(11, 23)]), (56, 68)
    if name == "identical":                                    # the same content in both frames: every color term is 0
        tex = SW.texture(rng, 60, 120)
        return [tex[:, :80].copy(), tex[:, 30:110].copy()], np.stack([T(1, 1), T(31, 1)]), (62, 112)
    if name == "flat":                                         # saturated flat bands: long runs of equal edges
        f = np.zeros((50, 70, 3), np.uint8)
        f[:, :, :] = 255
        f[20:30] = 0
        return [f, f.copy()], np.stack([T(1, 1), T(25, 1)]), (52, 96)
    if name == "contained":                                    # frame 1 inside frame 0
        frames = [rng.integers(0, 256, s + (3,), np.uint8) for s in ((40, 50), (14, 16))]
        return frames, np.stack([T(1, 1), T(17, 13)]), (42, 52)
    raise KeyError(name)


UNIQUE = ["noisy", "order", "clipped", "warped"]
TIES = ["identical", "flat"]


def _fed(name):
    frames, M, (Hc, Wc) = gc_case(name)
    return SM.fed(frames, M, Hc, Wc)


def _pairs_unique(imgs, masks, tls):
    """Every pair's minimum cut is unique on its intersection (as restate visits them)."""
    out = [m.copy() for m in masks]
    for i, j, rect in SM.pairs(tls, [m.shape for m in out]):
        lo, hi = GC.bounds(*GC.pair_graph(imgs, out, tls, i, j, rect))
        inner = (slice(GC.GAP, GC.GAP + rect[3] - rect[1]), slice(GC.GAP, GC.GAP + rect[2] - rect[0]))
        if not np.array_equal(lo[inner], hi[inner]):
            return False
        seams, _ = GC.restate([imgs[i], imgs[j]], [out[i], out[j]], [tls[i], tls[j]])
        out[i], out[j] = seams
    return True


@pytest.mark.parametrize("name", UNIQUE)
def test_restatement_equals_cv2_where_the_cut_is_unique(name):
    _, imgs, masks, tls = _fed(name)
    assert _pairs_unique(imgs, masks, tls)
    got, cuts = GC.restate(imgs, masks, tls)
    assert SL._equal(got, GC.cv2_seams(imgs, masks, tls))
    assert len(cuts) == len(SM.pairs(tls, [m.shape for m in masks])) and all(c > 0 for c in cuts)
    assert SL._equal(masks, _fed(name)[2])                    # the inputs are left alone


@pytest.mark.parametrize("name", TIES)
def test_cv2_lies_within_the_lattice_bounds_on_ties(name):
    _, imgs, masks, tls = _fed(name)
    (i, j, rect), = SM.pairs(tls, [m.shape for m in masks])
    lo, hi = GC.bounds(*GC.pair_graph(imgs, masks, tls, i, j, rect))
    x0, y0, x1, y1 = rect
    inner = (slice(GC.GAP, GC.GAP + y1 - y0), slice(GC.GAP, GC.GAP + x1 - x0))
    ref = GC.cv2_seams(imgs, masks, tls)
    vi = masks[i][y0 - tls[i][1]:y1 - tls[i][1], x0 - tls[i][0]:x1 - tls[i][0]] != 0
    vj = masks[j][y0 - tls[j][1]:y1 - tls[j][1], x0 - tls[j][0]:x1 - tls[j][0]] != 0
    kept_i = ref[i][y0 - tls[i][1]:y1 - tls[i][1], x0 - tls[i][0]:x1 - tls[i][0]] != 0
    both = vi & vj                                             # where both hold p, p in S exactly when frame i keeps it
    assert (kept_i[both] >= lo[inner][both]).all() and (kept_i[both] <= hi[inner][both]).all()
    assert (hi & ~lo).sum() > 100                              # a real tie: many pixels between the bounds
    got, _ = GC.restate(imgs, masks, tls)
    kept = got[i][y0 - tls[i][1]:y1 - tls[i][1], x0 - tls[i][0]:x1 - tls[i][0]] != 0
    assert np.array_equal(kept[both], hi[inner][both])         # the canonical cut: the largest source set


def test_visiting_order_changes_the_result():
    _, imgs, masks, tls = _fed("order")
    fwd, _ = GC.restate(imgs, masks, tls)
    perm = [2, 0, 1]
    rev, _ = GC.restate([imgs[k] for k in perm], [masks[k] for k in perm], [tls[k] for k in perm])
    back = [None] * 3
    for q, k in enumerate(perm):
        back[k] = rev[q]
    assert not SL._equal(back, fwd)


def test_a_contained_frame_vanishes():
    _, imgs, masks, tls = _fed("contained")
    got, cuts = GC.restate(imgs, masks, tls)
    assert SL._equal(got, GC.cv2_seams(imgs, masks, tls))
    assert not got[1].any() and (got[0] == masks[0]).all() and cuts == [0]


@pytest.mark.parametrize("side", ["no_source", "no_sink"])
def test_pairs_without_source_or_sink_pixels(side):
    """Frame j covers frame i's whole window (no source pixel) or the other way round (no sink pixel): the cut is 0 and
    the whole window is on the empty side's opposite."""
    rng = np.random.default_rng(4)
    big, small = rng.integers(0, 256, (40, 50, 3), np.uint8), rng.integers(0, 256, (12, 14, 3), np.uint8)
    frames, M = ([small, big], [T(17, 13), T(1, 1)]) if side == "no_source" else ([big, small], [T(1, 1), T(17, 13)])
    take, imgs, masks, tls = SM.fed(frames, np.stack(M), 42, 52)
    (i, j, rect), = SM.pairs(tls, [m.shape for m in masks])
    Tset, _, cut = GC.solve(*GC.pair_graph(imgs, masks, tls, i, j, rect))
    assert cut == 0 and (Tset.all() if side == "no_source" else not Tset.any())
    got, _ = GC.restate(imgs, masks, tls)
    assert SL._equal(got, GC.cv2_seams(imgs, masks, tls))


def test_capacity_and_certificate_on_scipys_flow():
    rng = np.random.default_rng(9)
    h, w = 7, 9
    hcap, vcap = rng.integers(1, 50, (h, w)), rng.integers(1, 50, (h, w))
    hcap[:, -1] = vcap[-1] = 0
    src = np.where(rng.random((h, w)) < 0.2, 100, 0)
    snk = np.where(rng.random((h, w)) < 0.2, 100, 0)
    Tset, lo, cut = GC.solve(hcap, vcap, src, snk)
    assert GC.capacity(~Tset, hcap, vcap, src, snk) == cut == GC.capacity(lo, hcap, vcap, src, snk)
    with pytest.raises(AssertionError):                        # an all-saturated residual is no certificate of this cut
        GC.check_certificate(hcap, vcap, src, snk, np.zeros((5, h, w), np.int64), Tset, cut)


# ---- the CLI ---------------------------------------------------------------------------------------------------------------
def test_cli_seam_flag():
    import mosaic_images as cli
    assert cli.build_parser().parse_args(["--frames", "raw", "--seam", "gc_color"]).seam == "gc_color"
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args(["--frames", "raw", "--seam", "gc_colour"])


def test_cli_mosaic_txt(tmp_path, monkeypatch):
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
                    gains=np.ones((3, 3)), last_ms=dict(prep=1.0, forward=2.0, blend=3.0, seam=0.25))

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
    argv = ["--frames", str(raw), "--out_dir", str(tmp_path / "out"), "--blend", "multiband", "--seam", "gc_color"]
    cli.run(cli.build_parser().parse_args(argv), None, lambda paths: None, lambda imgs: [b"jpeg"])
    txt = (tmp_path / "out" / "mosaic.txt").read_text().splitlines()
    assert seen == dict(seam="gc_color")
    assert txt[0] == "canvas 4 6 ref 1 blend multiband 5 seam gc_color"


def test_build_mosaic_takes_gc_color_and_still_rejects_graphcut():
    from unsuperviseddeephomographyral2018_b200 import mosaic
    assert "gc_color" in mosaic.SEAM and "graphcut" not in mosaic.SEAM
