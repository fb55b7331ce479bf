"""Host-side tests of the mosaic's exposure compensation: the NumPy restatement (oracle/exposure.py) against
cv2.detail_GainCompensator and ChannelsCompensator, apply against cv2's, the pair lists, the exact rounding of the
statistics kernel's fixed-point norm sums, mosaic_images.py's --compensate flags and mosaic.txt, and the compiled kernels
(no spills)."""
import math
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

cv2 = pytest.importorskip("cv2")
from oracle import exposure as EX  # noqa: E402


# ---- random ROI layouts --------------------------------------------------------------------------------------------------
def layout(seed, fill=0.8):
    """Fed images, masks and top-lefts: overlapping frames, a pair with no overlap, a pair whose rectangles meet but whose
    masks do not (N = 1), and an isolated frame (skipped, gain 1)."""
    rng = np.random.default_rng(seed)
    rects = [(0, 0, 40, 30), (20 + seed % 5, 10, 40, 30), (50, 25, 30, 20), (10, 35, 35, 25), (200, 200, 10, 10),
             (90, 0, 20, 20), (100, 5, 20, 20)]
    imgs, masks, tls = [], [], []
    for x, y, w, h in rects:
        base = rng.uniform(0.6, 1.4)
        imgs.append(np.clip(rng.integers(0, 200, (h, w, 3)) * base, 0, 255).astype(np.uint8))
        masks.append(np.where(rng.random((h, w)) < fill, 255, 0).astype(np.uint8))
        tls.append((x, y))
    masks[5][:, 10:] = 0                                       # frames 5 and 6 meet at x 100..110 but no pixel is set in both
    masks[6][:, :10] = 0
    return imgs, masks, tls


def _pair_keys(stats):
    return {(p["i"], p["j"]): p for p in stats}


@pytest.mark.parametrize("feeds", [1, 2, 3])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_layout_has_every_kind_of_pair(seed, feeds):
    imgs, masks, tls = layout(seed)
    st = _pair_keys(EX.pair_stats(imgs, masks, tls))
    assert (0, 5) not in st and (0, 4) not in st                # rectangles that do not intersect
    assert st[(5, 6)]["count"] == 0                            # rectangles meet, masks do not: N = 1
    assert st[(0, 1)]["count"] > 0 and st[(4, 4)]["count"] > 0
    g, _ = EX.restate(imgs, masks, tls, "gain", feeds)
    assert np.all(g[4] == 1.0) and np.all(g[5] == 1.0) and np.all(g[6] == 1.0)     # skipped
    assert np.all(g[:4] != 1.0)


@pytest.mark.parametrize("feeds", [1, 2, 3])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_channels_gains_equal_cv2_bit_for_bit(seed, feeds):
    imgs, masks, tls = layout(seed)
    ref, _ = EX.cv2_gains(imgs, masks, tls, "channels", feeds)
    got, _ = EX.restate(imgs, masks, tls, "channels", feeds)
    assert np.array_equal(got, ref)


@pytest.mark.parametrize("feeds", [1, 2, 3])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_gain_mode_equals_cv2_within_its_summation_error(seed, feeds):
    """cv2 adds the norms in row order; the kernel's sums are exact and rounded once.  With cv2's order the restatement
    gives cv2's gains; with the exact sums the gains move by no more than the gap between the two sums allows."""
    imgs, masks, tls = layout(seed)
    ref, _ = EX.cv2_gains(imgs, masks, tls, "gain", feeds)
    rows, _ = EX.restate(imgs, masks, tls, "gain", feeds, summation="rows")
    assert np.abs(rows / ref - 1).max() <= 4e-15
    exact, _ = EX.restate(imgs, masks, tls, "gain", feeds, summation="exact")
    # cv2's own summation error: the relative gap between its row-order sum and math.fsum of the same norms
    gap = 0.0
    for p, q in zip(EX.pair_stats(imgs, masks, tls, "rows"), EX.pair_stats(imgs, masks, tls, "exact")):
        for a, b in zip(p["norms"], q["norms"]):
            if b:
                gap = max(gap, abs(a - b) / b)
    assert gap > 0                                            # the two sums do differ here
    # the gains are a smooth function of the sums (the system's condition number is below 50 on these layouts): 100 x
    # the relative gap per feed bounds their move
    assert np.abs(exact / ref - 1).max() <= 100 * feeds * gap + 4e-15, (np.abs(exact / ref - 1).max(), gap)


def test_isolated_and_single_frames_keep_gain_1():
    imgs, masks, tls = layout(0)
    for k in (4, 5):
        g, _ = EX.cv2_gains([imgs[k]], [masks[k]], [tls[k]], "gain", 2)
        r, _ = EX.restate([imgs[k]], [masks[k]], [tls[k]], "gain", 2)
        assert np.all(g == 1.0) and np.all(r == 1.0)


# ---- apply -----------------------------------------------------------------------------------------------------------------
def test_apply_equals_cv2_with_ties_and_saturation():
    """rint of the float64 product, ties to even, saturated: 1.5 puts every odd value on a tie, 0.5 every odd value."""
    v = np.arange(256, dtype=np.uint8).reshape(16, 16, 1).repeat(3, 2)
    mask = np.full((16, 16), 255, np.uint8)
    for g in (1.5, 0.5, 1.0, 1.3, 0.75, 2.0, 0.9999999999999999, 1.0000000000000002, 0.0):
        c = EX.compensator("gain", 1)
        c.setMatGains([np.array([[g]])])
        assert np.array_equal(c.apply(0, (0, 0), v.copy(), mask), EX.apply(v, g)), g
        c = EX.compensator("channels", 1)
        gc = np.array([g, 1.25, 0.625])
        c.setMatGains([np.array([[gc[0]], [gc[1]], [gc[2]], [0.0]])])
        assert np.array_equal(c.apply(0, (0, 0), v.copy(), mask), EX.apply(v, gc)), g
    assert list(EX.apply(np.array([1, 3, 5, 171], np.uint8), 1.5)) == [2, 4, 8, 255]
    # float64, not float32: 95 x 0.3 is 28.499999999999996 in float64 (28) but 28.500002 in float32 (29); cv2 gives 28
    c = EX.compensator("gain", 1)
    c.setMatGains([np.array([[0.3]])])
    img = np.full((2, 2, 3), 95, np.uint8)
    assert c.apply(0, (0, 0), img.copy(), mask[:2, :2])[0, 0, 0] == EX.apply(img, 0.3)[0, 0, 0] == 28
    assert np.rint(np.float32(95) * np.float32(0.3)) == 29


# ---- pairs and the fixed-point norm sums ---------------------------------------------------------------------------------
def test_roi_pairs_with_the_diagonal_equal_the_oracle():
    from unsuperviseddeephomographyral2018_b200 import ops
    rng = np.random.default_rng(3)
    for _ in range(20):
        m = int(rng.integers(1, 30))
        x0, y0 = rng.integers(0, 200, m), rng.integers(0, 200, m)
        rois = np.stack([x0, y0, x0 + rng.integers(1, 60, m), y0 + rng.integers(1, 60, m)], 1)
        ptr, pj = ops.roi_pairs(rois, True)
        got = [(i, int(j)) for i in range(m) for j in pj[ptr[i]:ptr[i + 1]]]
        assert got == [(i, j) for i, j, _ in EX.pairs(rois.tolist())]


def _limbs(s):
    """A norm -> the kernel's fixed-point q = s 2^52 as three 21-bit limbs."""
    q = int(s * 2.0 ** 52)
    assert q == s * 2.0 ** 52 and q < 2 ** 61
    return q & 0x1FFFFF, (q >> 21) & 0x1FFFFF, q >> 42


def test_fixed_point_norm_sum_rounds_like_fsum():
    """Every norm is 0 or a multiple of 2^-52 below 2^9, so q is exact; the limb sums rounded once equal math.fsum."""
    from unsuperviseddeephomographyral2018_b200 import ops
    rng = np.random.default_rng(0)
    every = [math.sqrt(float(v)) for v in range(3 * 255 * 255 + 1)]
    for s in every:
        _limbs(s)
    for trial in range(40):
        n = int(rng.integers(1, 200000))
        if trial % 4 == 0:
            px = rng.integers(0, 256, (n, 3))
        elif trial % 4 == 1:
            px = rng.integers(0, 3, (n, 3))                     # small norms: 0, 1, sqrt 2, ...
        elif trial % 4 == 2:
            px = np.full((n, 3), 255) - rng.integers(0, 2, (n, 3))
        else:
            px = rng.integers(0, 256, (n, 1)).repeat(3, 1)
        s = [every[v] for v in (px.astype(np.int64) ** 2).sum(1)]
        tot = [0, 0, 0]
        for v in s:
            for k, l in enumerate(_limbs(v)):
                tot[k] += l
        assert ops.exposure_norm_sum(*tot) == math.fsum(s)
    # the largest sums the kernel takes: 2^31 pixels of the largest norm, and a total whose rounding is a tie
    big = math.sqrt(3 * 255 * 255)
    l = _limbs(big)
    assert ops.exposure_norm_sum(*[v * 2 ** 31 for v in l]) == big * 2 ** 31
    assert ops.exposure_norm_sum(1, 0, 2 ** 11) == 2.0 == math.fsum([2.0, 2.0 ** -52])      # (2^53 + 1) 2^-52: a tie, to even


# ---- the CLI ---------------------------------------------------------------------------------------------------------------
def test_cli_compensate_flags():
    import mosaic_images as cli
    a = cli.build_parser().parse_args(["--frames", "raw"])
    assert (a.compensate, a.compensate_feeds) == ("none", 1)
    a = cli.build_parser().parse_args(["--frames", "raw", "--compensate", "channels", "--compensate_feeds", "3"])
    assert (a.compensate, a.compensate_feeds) == ("channels", 3)
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args(["--frames", "raw", "--compensate", "blocks"])
    for feeds in (0, 17):
        with pytest.raises(SystemExit):
            cli.run(cli.build_parser().parse_args(["--frames", "raw", "--compensate", "gain", "--compensate_feeds", str(feeds)]),
                    None, None, None)


@pytest.mark.parametrize("compensate", ["none", "gain", "channels"])
def test_cli_mosaic_txt(tmp_path, monkeypatch, compensate):
    """Without compensation mosaic.txt is the parent's format; with it the first line ends in ` compensate MODE F` and each
    frame line in its three gains as %.17g (they read back to the same doubles)."""
    import torch
    import mosaic_images as cli
    from unsuperviseddeephomographyral2018_b200 import mosaic
    raw = tmp_path / "raw"
    raw.mkdir()
    for k in range(3):
        (raw / ("F_%d.JPG" % k)).write_bytes(b"")
    seen = {}
    gains = np.array([[1.0 / 3, 0.1, 1.0], [1.0, 1.0, 1.0], [1.2345678901234567, 2.0 / 3, 0.9]])

    def fake_build(est, imgs, ref, refine, feather, float32_M=False, blend="feather", bands=5, **kw):
        seen.update(kw)
        M = np.stack([np.array([[1.0, 0, 10.0 * k], [0, 1.0, 0.5], [0, 0, 1.0]]) for k in range(3)])
        return dict(mosaic=torch.zeros(4, 6, 3, dtype=torch.uint8), mask=torch.zeros(4, 6, dtype=torch.uint8), M=M,
                    kept=np.array([True, False, True]), ref=1, H_pairs=np.stack([np.eye(3)] * 2), refine=None, gains=gains,
                    last_ms=dict(prep=1.0, forward=2.0, blend=3.0, **(dict(compensate=0.25) if kw else {})))

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
    argv = ["--frames", str(raw), "--out_dir", str(tmp_path / "out"), "--blend", "multiband"]
    if compensate != "none":
        argv += ["--compensate", compensate, "--compensate_feeds", "2"]
    cli.run(cli.build_parser().parse_args(argv), None, lambda paths: None, lambda imgs: [b"jpeg"])
    txt = (tmp_path / "out" / "mosaic.txt").read_text().splitlines()
    if compensate == "none":
        assert seen == {}
        assert txt[0] == "canvas 4 6 ref 1 blend multiband 5"
        assert txt[1] == "F_0.JPG kept 1 0 0 0 1 0.5 0 0 1"
        return
    assert seen == dict(compensate=compensate, compensate_feeds=2)
    assert txt[0] == "canvas 4 6 ref 1 blend multiband 5 compensate %s 2" % compensate
    for k, ln in enumerate(txt[1:]):
        parts = ln.split()
        assert len(parts) == 2 + 9 + 3
        assert np.array_equal(np.array([float(v) for v in parts[11:]]), gains[k])
    assert txt[1].startswith("F_0.JPG kept 1 0 0 0 1 0.5 0 0 1 ")


# ---- the compiled kernels -----------------------------------------------------------------------------------------------
def _tool(name):
    p = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), name)
    return p if os.path.exists(p) else shutil.which(name)


@pytest.mark.skipif(_tool("nvcc") is None, reason="the CUDA toolkit is not installed")
def test_exposure_stats_and_gain_blend_kernels_do_not_spill(tmp_path):
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
        if m and current and re.search(r"exposure_|invert_kernelINS_13ExposureFrame|mosaic_blend_u8_kernelILi\dELb1ELb0ELb0E|"
                                       r"multiband_base_kernelILb0E", current):
            seen[current] = tuple(int(v) for v in m.groups())
    assert len(seen) == 5, seen                               # stats, inverses, blend C = 1 and 3, the multi-band base
    assert all(v == (0, 0, 0) for v in seen.values()), seen
