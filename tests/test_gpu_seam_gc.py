"""GPU tests of the graph-cut seams: udh_debug_grid_mincut against scipy (cut value and T byte for byte) on random and
maze grids, its residuals certified at full size (every pair of a 6-frame 1080 x 1920 sweep, the 12 MP pair's window),
udh_mosaic_seam_gc_masks_u8 against oracle/seam_gc.restate and cv2, both blends with graph-cut seams against their
oracles, run independence, the buffer contract, mosaic_images.py --seam gc_color, and the quality check against the
Voronoi assignment."""
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
import test_seam_gc_logic as GL  # noqa: E402
import test_seam_logic as SL  # noqa: E402
from oracle import seam as SM  # noqa: E402
from oracle import seam_gc as GC  # noqa: E402

pytestmark = pytest.mark.gpu
T = SL.T


def _ops():
    from unsuperviseddeephomographyral2018_b200 import ops
    return ops


def _mincut(hcap, vcap, src, snk, residual=False):
    d = [torch.from_numpy(np.ascontiguousarray(a, np.int32)).cuda() for a in (hcap, vcap, src, snk)]
    out = _ops().grid_mincut(*d, residual=residual)
    return {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in out.items()}


# ---- the min-cut core ------------------------------------------------------------------------------------------------------
def random_grid(rng, h, w, cap, terms):
    hcap = rng.integers(1, cap + 1, (h, w)) if cap > 1 else np.ones((h, w), np.int64)
    vcap = rng.integers(1, cap + 1, (h, w)) if cap > 1 else np.ones((h, w), np.int64)
    hcap[:, -1] = 0
    vcap[-1] = 0
    src = np.where(rng.random((h, w)) < 0.1, GC.TERM, 0) if terms in ("both", "source") else np.zeros((h, w), np.int64)
    snk = np.where(rng.random((h, w)) < 0.1, GC.TERM, 0) if terms in ("both", "sink") else np.zeros((h, w), np.int64)
    if terms == "both":
        src[0, 0], snk[-1, -1] = GC.TERM, GC.TERM
    return hcap, vcap, src, snk


SIZES = [(1, 1), (1, 57), (61, 1), (31, 33), (32, 32), (33, 65), (97, 130), (257, 300)]


@pytest.mark.parametrize("terms", ["both", "none", "source", "sink"])
@pytest.mark.parametrize("cap", [1, 391151, 50000])
@pytest.mark.parametrize("h,w", SIZES)
def test_grid_mincut_equals_scipy(h, w, cap, terms):
    rng = np.random.default_rng(h * 1000 + w + cap + len(terms))
    g = random_grid(rng, h, w, cap, terms)
    Tset, _, cut = GC.solve(*g)
    got = _mincut(*g)
    assert got["cut"] == cut
    assert np.array_equal(got["T"], Tset.astype(np.uint8))


def maze(n):
    """An n x n maze: a one-pixel corridor along every even row, joined to the next at alternate ends (capacity 5 along
    it, 0 across its walls), the source at one end and the sink at the other, so every augmenting path is about n^2 / 2
    long."""
    hcap = np.zeros((n, n), np.int64)
    vcap = np.zeros((n, n), np.int64)
    rows = list(range(0, n, 2))
    for q, y in enumerate(rows):
        hcap[y, :n - 1] = 5
        if q + 1 < len(rows):
            x = n - 1 if q % 2 == 0 else 0
            vcap[y, x] = vcap[y + 1, x] = 5
    src, snk = np.zeros((n, n), np.int64), np.zeros((n, n), np.int64)
    src[0, 0] = GC.TERM
    snk[rows[-1], n - 1 if len(rows) % 2 == 0 else 0] = GC.TERM
    return hcap, vcap, src, snk, len(rows) * n + len(rows) - 1


@pytest.mark.parametrize("n", [40, 101])
def test_grid_mincut_on_a_maze(n):
    hcap, vcap, src, snk, length = maze(n)
    assert length > n * n // 3
    Tset, _, cut = GC.solve(hcap, vcap, src, snk)
    got = _mincut(hcap, vcap, src, snk, residual=True)
    assert got["cut"] == cut == 5 and np.array_equal(got["T"], Tset.astype(np.uint8))
    GC.check_certificate(hcap, vcap, src, snk, got["residual"], got["T"] != 0, got["cut"])


# ---- certificates at full size ---------------------------------------------------------------------------------------------
def _certify_pairs(name):
    frames, M, (Hc, Wc) = GS.case(name)
    _, imgs, masks, tls = SM.fed(frames, M, Hc, Wc)
    n = 0
    for i, j, rect in SM.pairs(tls, [m.shape for m in masks]):
        g = GC.pair_graph(imgs, masks, tls, i, j, rect)
        got = _mincut(*g, residual=True)
        GC.check_certificate(*g, got["residual"], got["T"] != 0, got["cut"])
        n += 1
    return n


@pytest.mark.parametrize("name", ["sweep1080", "pair12mp"])
def test_certificate_at_full_size(name):
    assert _certify_pairs(name) >= 1


# ---- seams ---------------------------------------------------------------------------------------------------------------------
def _gpu_seams(frames, M, Hc, Wc):
    return _ops().mosaic_seam_masks(GS._cuda(frames), M, Hc, Wc, finder="gc_color")


@pytest.mark.parametrize("name", GL.UNIQUE + GL.TIES + ["contained"])
def test_seams_equal_the_restatement(name):
    frames, M, (Hc, Wc) = GL.gc_case(name)
    got = _gpu_seams(frames, M, Hc, Wc)
    take, imgs, masks, tls = SM.fed(frames, M, Hc, Wc)
    assert got["take"] == take
    ref, cuts = GC.restate(imgs, masks, tls)
    assert [int(c) for c in got["cut"]] == cuts
    for k, (s, b, rs, rb) in enumerate(zip(got["seam"], got["blend"], ref, SM.blend_masks(ref, masks))):
        assert np.array_equal(s.cpu().numpy(), rs), ("seam", k)
        assert np.array_equal(b.cpu().numpy(), rb), ("blend", k)
    if name in GL.UNIQUE:
        assert SL._equal([s.cpu().numpy() for s in got["seam"]], GC.cv2_seams(imgs, masks, tls))


def test_two_runs_are_bit_identical():
    frames, M, (Hc, Wc) = GS.case("sweep1080")
    a, b = _gpu_seams(frames, M, Hc, Wc), _gpu_seams(frames, M, Hc, Wc)
    assert np.array_equal(a["cut"], b["cut"])
    assert all(np.array_equal(x.cpu().numpy(), y.cpu().numpy()) for x, y in zip(a["seam"] + a["blend"], b["seam"] + b["blend"]))


def _blend_masks(frames, M, Hc, Wc):
    rgb = [f if f.ndim == 3 and f.shape[2] == 3 else np.repeat(f.reshape(f.shape[0], f.shape[1], 1), 3, 2) for f in frames]
    s = _gpu_seams(rgb, M, Hc, Wc)
    out = [None] * len(frames)
    for q, b in zip(s["take"], s["blend"]):
        out[q] = b
    return out


@pytest.mark.parametrize("gains", [False, True])
@pytest.mark.parametrize("name", ["order", "warped"])
def test_multiband_with_gc_seams_equals_the_oracle(name, gains):
    frames, M, (Hc, Wc) = GL.gc_case(name)
    g = np.random.default_rng(7).uniform(0.6, 1.5, (len(frames), 3)) if gains else None
    out, mask = _ops().mosaic_multiband_u8(GS._cuda(frames), M, Hc, Wc, 5, gains=g, masks=_blend_masks(frames, M, Hc, Wc))
    ref, ref_mask = GC.multiband(frames, M, Hc, Wc, 5, g)
    assert np.array_equal(mask.cpu().numpy(), ref_mask) and np.array_equal(out.cpu().numpy(), ref)


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("name", ["clipped", "warped"])
def test_feathered_blend_with_gc_seams_equals_the_oracle(name, C):
    frames, M, (Hc, Wc) = GL.gc_case(name)
    frames = [f[..., :C].copy() for f in frames]
    out, mask = _ops().mosaic_blend_u8(GS._cuda(frames), M, Hc, Wc, 64, masks=_blend_masks(frames, M, Hc, Wc))
    ref, ref_mask = GC.feather(frames, M, Hc, Wc, 64)
    assert np.array_equal(mask.cpu().numpy(), ref_mask) and np.array_equal(out.cpu().numpy(), ref)


# ---- the buffer contract ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(1, 1), (7, 33), (45, 31), (70, 97)])
def test_grid_mincut_under_both_poisons(monkeypatch, h, w):
    g = random_grid(np.random.default_rng(h + w), h, w, 391151, "both")
    Tset, _, cut = GC.solve(*g)

    def inputs(fr, p):
        return tuple(BC.framed_input(fr, p, np.ascontiguousarray(a, np.int32), name=n) for a, n in zip(g, ("hcap", "vcap", "src", "snk")))
    # the residuals are left out: the flow races, only the cut is unique
    res = BC.under_both_poisons(monkeypatch, [_ops()], lambda fr, p, *a: _ops().grid_mincut(*a), inputs)[0]
    assert res["cut"] == cut and np.array_equal(res["T"], Tset.astype(np.uint8))


@pytest.mark.parametrize("name", ["clipped", "order"])
def test_seam_gc_under_both_poisons(monkeypatch, name):
    frames, M, (Hc, Wc) = GL.gc_case(name)
    _, imgs, masks, tls = SM.fed(frames, M, Hc, Wc)
    ref, cuts = GC.restate(imgs, masks, tls)

    def inputs(fr, p):
        return tuple(BC.framed_input(fr, p, f, name="frame%d" % k) for k, f in enumerate(frames))
    res = BC.under_both_poisons(monkeypatch, [_ops()], lambda fr, p, *f: _ops().mosaic_seam_masks(list(f), M, Hc, Wc, finder="gc_color"),
                                inputs)[0]
    assert SL._equal(res["seam"], ref) and [int(c) for c in res["cut"]] == cuts


# ---- build_mosaic and the CLI ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("blend", ["feather", "multiband"])
def test_build_mosaic_with_gc_seams(blend):
    from unsuperviseddeephomographyral2018_b200 import mosaic
    _, frames, _, H = SW.sweep(3, 100, 130, seed=3)
    c = mosaic.build_mosaic(GS.TrueEstimator(H), GS._cuda(frames), blend=blend, seam="gc_color")
    Hc, Wc = c["mask"].shape
    ref = GC.multiband(frames, c["M"], Hc, Wc, 5)[0] if blend == "multiband" else GC.feather(frames, c["M"], Hc, Wc, 64)[0]
    assert c["last_ms"]["seam"] > 0 and np.array_equal(c["mosaic"].cpu().numpy(), ref)


def test_cli_end_to_end(tmp_path):
    import mosaic_images as cli
    raw = tmp_path / "raw"
    raw.mkdir()
    _, frames, _, _ = SW.sweep(3, 160, 200, seed=9)
    names = ["DSC_%04d.JPG" % k for k in range(3)]
    for nm, f in zip(names, frames):
        cv2.imwrite(str(raw / nm), f[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, 95])
    out = tmp_path / "mosaic"
    assert cli.main(["--frames", str(raw), "--out_dir", str(out), "--seeded_weights", "True", "--model_dir", str(tmp_path / "none"),
                     "--blend", "multiband", "--seam", "gc_color"]) == 0
    txt = (out / "mosaic.txt").read_text().splitlines()
    head = txt[0].split()
    assert head[5:] == ["blend", "multiband", "5", "seam", "gc_color"]
    Hc, Wc = int(head[1]), int(head[2])
    imgs, Ms = [], []
    for ln, nm in zip(txt[1:], names):
        parts = ln.split()
        if parts[1] == "kept":
            imgs.append(cv2.imread(str(raw / nm))[..., ::-1].copy())
            Ms.append(np.array([float(v) for v in parts[2:11]]).astype(np.float32).astype(np.float64).reshape(3, 3))
    mos, _ = GC.multiband(imgs, np.stack(Ms), Hc, Wc, 5)
    assert (out / "mosaic.jpg").read_bytes() == _ops().encode_jpeg(np.ascontiguousarray(mos[..., ::-1])[None])[0]


# ---- quality ------------------------------------------------------------------------------------------------------------------
def test_gc_cuts_beat_the_voronoi_assignment_on_a_drifting_sweep():
    """test_gpu_seam's drifting sweep: every pair's graph-cut value equals scipy's on the oracle's window graph and is at
    most the capacity of the Voronoi labelling of the same window and masks (d_i < d_j: source side); both seamed
    mosaics' mean absolute difference to the true texture over the overlaps is reported."""
    from unsuperviseddeephomographyral2018_b200 import mosaic
    tex, frames, A, H = SW.sweep(6, 480, 640, seed=11)
    rng = np.random.default_rng(11)
    Hp = np.stack([T(*rng.uniform(-3, 3, 2)) @ h for h in H])
    G, r = mosaic.chain_to_reference(Hp)
    M, (Hc, Wc), kept = mosaic.canvas([f.shape[:2] for f in frames], G, r)
    got = _gpu_seams(frames, M, Hc, Wc)
    _, imgs, masks, tls = SM.fed(frames, M, Hc, Wc)
    cur = [m.copy() for m in masks]
    for q, (i, j, rect) in enumerate(SM.pairs(tls, [m.shape for m in cur])):
        g = GC.pair_graph(imgs, cur, tls, i, j, rect)
        si, sj = SM._window(cur[i], tls[i], *rect), SM._window(cur[j], tls[j], *rect)
        both = si & sj
        vor = SM.l1_distance(si & ~both) < SM.l1_distance(sj & ~both)
        assert int(got["cut"][q]) == GC.solve(*g)[2]              # the device-built window is the oracle's graph
        assert int(got["cut"][q]) <= GC.capacity(vor, *g)
        seams, _ = GC.restate([imgs[i], imgs[j]], [cur[i], cur[j]], [tls[i], tls[j]])
        cur[i], cur[j] = seams
    seen = cv2.warpPerspective(tex, A[r] @ np.linalg.inv(M[r]), (Wc, Hc), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP)
    cover = np.zeros((Hc, Wc), np.int32)
    for m, (x, y) in zip(masks, tls):
        cover[y:y + m.shape[0], x:x + m.shape[1]] += m != 0
    over = cover >= 2
    res = {}
    for label, finder in (("voronoi", "voronoi"), ("gc_color", "gc_color")):
        s = _ops().mosaic_seam_masks(GS._cuda(frames), M, Hc, Wc, finder=finder)
        bm = [None] * len(frames)
        for q, b in zip(s["take"], s["blend"]):
            bm[q] = b
        for blend in ("multiband", "feather"):
            if blend == "multiband":
                out, _ = _ops().mosaic_multiband_u8(GS._cuda(frames), M, Hc, Wc, 5, masks=bm)
            else:
                out, _ = _ops().mosaic_blend_u8(GS._cuda(frames), M, Hc, Wc, 64, masks=bm)
            res[(label, blend)] = float(np.abs(out.cpu().numpy().astype(np.int32) - seen.astype(np.int32))[over].mean())
    print("drifting sweep, overlap MAD to the texture: " + ", ".join("%s %s %.3f" % (k[0], k[1], v) for k, v in res.items()))
    assert all(np.isfinite(v) for v in res.values())
