"""Host-side tests of the mosaic's block exposure compensation: the NumPy restatement (oracle/exposure_blocks.py) against
cv2.detail_BlocksGainCompensator and BlocksChannelsCompensator (maps bit for bit, apply'd bytes within the resize's
near-tie bound), the analytic block-pair list and the sparse assembly against cv2-order dense assembly, the resize taps,
mosaic_images.py's flags, and the compiled kernels (no spills)."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

cv2 = pytest.importorskip("cv2")
import test_seam_logic as SL  # noqa: E402
from oracle import exposure as EX  # noqa: E402
from oracle import exposure_blocks as XB  # noqa: E402


def vignette(img, strength, gain):
    """img scaled by gain and a radial falloff of `strength` at the corners (uint8)."""
    h, w = img.shape[:2]
    yy, xx = np.mgrid[0:h, 0:w]
    r2 = ((xx - (w - 1) / 2.0) / (w / 2.0)) ** 2 + ((yy - (h - 1) / 2.0) / (h / 2.0)) ** 2
    return np.clip(img * (gain * (1 - strength * r2 / 2))[..., None], 0, 255).astype(np.uint8)


def fed_case(name):
    """(imgs, masks, tls) as the compensators are fed."""
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "pairs":                       # sides that are not block multiples, an exposure step, vignetting; frames 3, 4
        rects = [(0, 0, 90, 70), (40, 10, 100, 61), (100, 5, 77, 50), (300, 300, 20, 20), (180, 0, 20, 20), (190, 0, 20, 20)]
        gains = [1.0, 0.7, 1.25, 1.0, 0.9, 1.1]
        imgs, masks, tls = [], [], []
        for (x, y, w, h), g in zip(rects, gains):
            imgs.append(vignette(rng.integers(40, 220, (h, w, 3)).astype(np.float64), 0.3, g))
            m = np.full((h, w), 255, np.uint8)
            m[:3, :5] = 0
            masks.append(m)
            tls.append((x, y))
        masks[4][:, 10:] = 0                  # frames 4 and 5 meet at x 190..200 but share no valid pixel: N = 1
        masks[5][:, :10] = 0
        return imgs, masks, tls
    frames, M, (Hc, Wc) = SL.frame_case(name)
    frames = [vignette(f.astype(np.float64), 0.3, g) for f, g in zip(frames, [1.0, 0.75, 1.2, 0.9, 1.1])]
    _, imgs, masks, tls = EX.fed(frames, M, Hc, Wc)
    return imgs, masks, tls


CASES = ["pairs", "clipped", "warped", "sweep"]


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


@pytest.mark.parametrize("feeds", [1, 2, 3])
@pytest.mark.parametrize("block", [16, 32, 48])
@pytest.mark.parametrize("mode", ["gain", "channels"])
@pytest.mark.parametrize("name", CASES)
def test_restated_maps_equal_cv2_bit_for_bit(name, mode, block, feeds):
    imgs, masks, tls = fed_case(name)
    ref, applied = XB.cv2_maps(imgs, masks, tls, mode, feeds, block)
    got, _, grids, _ = XB.restate(imgs, masks, tls, mode, feeds, block)
    assert len(got) == len(ref)
    for a, b in zip(got, ref):
        assert _bits_equal(a, b)
    # the apply'd bytes: equal, or off by one where the resize's float32 rounding can move float32(v) g across a tie
    for img, mp, cv in zip(imgs, got, applied):
        mine = XB.apply_map(img, mp)
        diff = mine != cv
        if diff.any():
            dg = XB.resize_gap(mp, img.shape[0], img.shape[1])
            assert (np.abs(mine.astype(int) - cv)[diff] == 1).all()
            assert XB.near_tie(img, mp, dg)[diff].all()


def test_isolated_frames_get_unit_maps_and_zero_count_pairs_add_beta():
    imgs, masks, tls = fed_case("pairs")
    maps, g, grids, trace = XB.restate(imgs, masks, tls, "gain", 1, 32)
    assert (maps[3] == 1).all() and (maps[4] == 1).all() and (maps[5] == 1).all()
    bi, bm, bt, _ = XB.blocks(imgs, masks, tls, 32, 32)
    o4 = sum(gx * gy for gx, gy, _, _ in grids[:4])
    zero = [p for p in trace[0] if p["i"] >= o4 and p["i"] != p["j"]]
    assert zero and all(p["count"] == 0 for p in zero)          # rectangles meet, masks do not
    # blocks without overlap (gain 1) sit next to solved blocks, and the filter spreads the solved gains into them
    first = g[:grids[0][0] * grids[0][1], 0]
    assert (first == 1).any() and (first != 1).any()
    assert (maps[0] != 1).all()


def test_block_grid_is_cv2s():
    from unsuperviseddeephomographyral2018_b200 import ops
    rois = np.array([[0, 0, 90, 70], [3, 4, 3 + 100, 4 + 61], [0, 0, 33, 17], [5, 5, 6, 6]])
    for block in (16, 32, 48):
        blocks, boff = ops.exposure_block_grid(rois, block)
        for r, b in zip(rois, blocks):
            assert tuple(int(v) for v in b) == XB.grid(r[3] - r[1], r[2] - r[0], block, block)[2:] + XB.grid(r[3] - r[1], r[2] - r[0], block, block)[:2]
        assert boff[-1] == sum(int(b[2]) * int(b[3]) for b in blocks)


@pytest.mark.parametrize("block", [16, 32, 48])
@pytest.mark.parametrize("name", CASES)
def test_block_pairs_and_sparse_system_equal_cv2_order_dense_assembly(name, block):
    """The analytic block-pair list is every pair of blocks whose rectangles intersect (an O(m^2) scan of the block
    corners); the CSR rows equal the dense A and b built in cv2's loop order, bit for bit, from the same statistics."""
    from unsuperviseddeephomographyral2018_b200 import ops
    imgs, masks, tls = fed_case(name)
    rois = np.array([(x, y, x + m.shape[1], y + m.shape[0]) for (x, y), m in zip(tls, masks)])
    blocks, boff = ops.exposure_block_grid(rois, block)
    cells = ops.exposure_block_cells(rois, blocks, boff)
    bi, bm, bt, _ = XB.blocks(imgs, masks, tls, block, block)
    brects = [(x, y, x + m.shape[1], y + m.shape[0]) for (x, y), m in zip(bt, bm)]
    want = [(i, j) for i, j, _ in EX.pairs(brects)]
    got = list(zip(cells["a"].tolist(), cells["b"].tolist()))
    assert sorted(got) == want
    assert len(set(cells["slot"].tolist())) == len(got)                       # one cell per block pair
    assert cells["slot"].max() < cells["nslots"]
    for mode in ("gain", "channels"):
        st = {(p["i"], p["j"]): p for p in EX.pair_stats(bi, bm, bt, "rows")}
        cnt = np.array([st[k]["count"] for k in got])
        chans = [("norms", None)] if mode == "gain" else [("sums", c) for c in range(3)]
        for key, c in chans:
            sa = np.array([st[k][key][0] if c is None else st[k][key][0, c] for k in got])
            sb = np.array([st[k][key][1] if c is None else st[k][key][1, c] for k in got])
            keep, ptr, col, val, rhs = ops.exposure_block_system(len(bi), cells["a"], cells["b"], cnt, sa, sb)
            A, b, kref = _dense(len(bi), st, key, c)
            assert np.array_equal(keep, kref)
            dense = np.zeros_like(A)
            for r in range(len(keep)):
                dense[r, col[ptr[r]:ptr[r + 1]]] = val[ptr[r]:ptr[r + 1]]
                assert (np.diff(col[ptr[r]:ptr[r + 1]]) > 0).all()
            assert np.array_equal(dense.view(np.uint64), A.view(np.uint64))
            assert np.array_equal(rhs.view(np.uint64), b.view(np.uint64))


def _dense(m, st, key, c):
    """cv2's dense system (oracle/exposure.solve's loop) -> (A, b, kept indices)."""
    N = np.zeros((m, m), np.int64)
    I = np.zeros((m, m))
    skip = np.ones(m, bool)
    for (i, j), p in st.items():
        N[i, j] = N[j, i] = max(1, p["count"])
        if p["count"] == 0:
            continue
        if i != j:
            skip[i] = skip[j] = False
        s1, s2 = (p[key][0], p[key][1]) if c is None else (p[key][0, c], p[key][1, c])
        I[i, j], I[j, i] = float(s1) / N[i, j], float(s2) / N[i, j]
    keep = np.flatnonzero(~skip)
    A = np.zeros((len(keep), len(keep)))
    b = np.zeros(len(keep))
    for ki, i in enumerate(keep):
        for kj, j in enumerate(keep):
            b[ki] += EX.BETA * int(N[i, j])
            A[ki, ki] += EX.BETA * int(N[i, j])
            if j != i:
                A[ki, ki] += 2 * EX.ALPHA * float(I[i, j]) * float(I[i, j]) * int(N[i, j])
                A[ki, kj] -= 2 * EX.ALPHA * float(I[i, j]) * float(I[j, i]) * int(N[i, j])
    return A, b, keep


def test_map_taps_are_the_restated_resize():
    from unsuperviseddeephomographyral2018_b200 import ops
    rng = np.random.default_rng(0)
    for (h, w), (H, W) in [((3, 3), (70, 90)), ((34, 60), (1080, 1920)), ((1, 4), (17, 100)), ((5, 6), (5, 6)), ((2, 2), (3, 2))]:
        mp = rng.uniform(0.5, 1.5, (h, w)).astype(np.float32)
        ct, rt = ops.map_taps(w, W), ops.map_taps(h, H)
        a0, a1 = ct[:, 2].view(np.float32), ct[:, 3].view(np.float32)
        b0, b1 = rt[:, 2].view(np.float32), rt[:, 3].view(np.float32)
        hr = mp[:, ct[:, 0]] * a0 + mp[:, ct[:, 1]] * a1
        got = hr[rt[:, 0]] * b0[:, None] + hr[rt[:, 1]] * b1[:, None]
        assert _bits_equal(got, XB.resize_map(mp, H, W))


def test_filter_is_the_symmetric_form():
    """One pass is (a + c) 1/4 + b 1/2, row then column; summing the three terms left to right differs."""
    rng = np.random.default_rng(1)
    mp = rng.uniform(0.5, 1.5, (7, 9)).astype(np.float32)
    k = np.array([[0.25, 0.5, 0.25]], np.float32)
    ref = cv2.sepFilter2D(mp, cv2.CV_32F, k, k)
    assert _bits_equal(XB.filter_pass(mp), ref)
    for shape in [(1, 1), (1, 5), (4, 1), (2, 3)]:
        m = rng.uniform(0.5, 1.5, shape).astype(np.float32)
        assert _bits_equal(XB.filter_pass(m), cv2.sepFilter2D(m, cv2.CV_32F, k, k).reshape(shape))


def test_cli_block_flags():
    import mosaic_images as cli
    args = cli.build_parser().parse_args(["--frames", "raw", "--compensate", "gain_blocks", "--compensate_block", "48"])
    assert args.compensate == "gain_blocks" and args.compensate_block == 48
    assert cli.build_parser().parse_args(["--frames", "raw", "--compensate", "channels_blocks"]).compensate_block == 32
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args(["--frames", "raw", "--compensate", "blocks"])


def test_build_mosaic_rejects_other_modes():
    from unsuperviseddeephomographyral2018_b200 import mosaic
    assert "gain_blocks" in mosaic.COMPENSATE and "channels_blocks" in mosaic.COMPENSATE


def test_block_and_gain_map_kernels_do_not_spill(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc) and not shutil.which("nvcc"):
        pytest.skip("nvcc not available")
    src = os.path.join(ROOT, "unsuperviseddeephomographyral2018_b200", "csrc", "warp_perspective.cu")
    out = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I", os.path.join(ROOT, "include"),
                          "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "wp.o")],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    blocks = re.split(r"Compiling entry function '", out.stderr)
    seen = 0
    for b in blocks:
        name = b.split("'")[0]
        if "gainblock" in name or "ExposureBlockFrame" in name or re.search(r"mosaic_blend_u8_kernelILi\dELb0ELb[01]ELb1E|"
                                                                             r"multiband_base_kernelILb1E", name):
            seen += 1
            assert "0 bytes spill stores, 0 bytes spill loads" in b, (name, b)
    assert seen >= 8
