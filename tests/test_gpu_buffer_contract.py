"""GPU tests of the buffer contract (tests/_buffer_contract.py): every entry point at the ragged sizes around its tiles runs
twice, with every workspace, output and input frame poisoned 0xFF and then 0x00; both runs must be bit-identical (no stale
read), equal the oracle the kernel's own tests use (no skipped element) and leave every 4096-byte frame intact (no write
past an end).  Inputs are framed by the run's poison, so a read past one changes a result.  Objects that keep a workspace
across calls (_ExposureStats, _ExposureBlockStats) have it re-poisoned between calls; JpegPlan keeps none (each decode
allocates its own).  Results carrying floating-point atomics (the photometric sums and dH, h4p_loss's metrics) are
compared within their run-to-run envelope instead of bit for bit.  Last, the CNN engine's workspace: an engine whose
workspace was all 0xFF before its initialisation steps as an untouched one does (bit for bit where the step is
deterministic, within the atomics' envelope from a shared state where it is not).

Not framed: the host-built tables ops copies with torch.from_numpy(...).to(dev) (tile lists, pair lists, ROI tables), the
engine's slab scratch, and the multi-GPU multicast path."""
import contextlib
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
from oracle import draw as D  # noqa: E402
from oracle import ecc as E  # noqa: E402
from oracle import exposure as EX  # noqa: E402
from oracle import exposure_blocks as XB  # noqa: E402
from oracle import gen_data as OG  # noqa: E402
from oracle import jpeg as J  # noqa: E402
from oracle import jpeg_enc as JE  # noqa: E402
from oracle import mosaic as OM  # noqa: E402
from oracle import multiband as MB  # noqa: E402
from oracle import png as PNG  # noqa: E402
from oracle import real as R  # noqa: E402
from oracle import resize as Z  # noqa: E402
from oracle import seam as SM  # noqa: E402
from oracle import warp_perspective as WP  # noqa: E402

pytestmark = pytest.mark.gpu
IN = BC.framed_input


def _ops():
    from unsuperviseddeephomographyral2018_b200 import ops
    return ops


def run(monkeypatch, call, inputs=None, same=BC.bit_equal, mods=None):
    """The result of call under both poisons (tests/_buffer_contract.under_both_poisons), ops' torch shimmed."""
    return BC.under_both_poisons(monkeypatch, mods or [_ops()], call, inputs, same)[0]


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def close(rtol):
    """same= for results with floating-point atomics: equal shapes and dtypes, all finite, each float array within rel L2
    rtol of the other; everything else bit-identical."""
    def same(a, b, where="out"):
        if isinstance(a, (list, tuple)):
            assert len(a) == len(b), where
            for k, (x, y) in enumerate(zip(a, b)):
                same(x, y, "%s[%d]" % (where, k))
        elif isinstance(a, np.ndarray) and a.dtype.kind == "f":
            assert a.shape == b.shape and a.dtype == b.dtype and np.isfinite(a).all() and np.isfinite(b).all(), where
            assert rel_l2(a, b) <= rtol, (where, rel_l2(a, b))
        else:
            BC.bit_equal(a, b, where)
    return same


def T(dx, dy):
    return np.array([[1.0, 0, dx], [0, 1.0, dy], [0, 0, 1.0]])


# ---- warps, gray, resizes ---------------------------------------------------------------------------------------------------
# dh * dw * C = 1, 2, 3 mod 4 and 0; 1x1, 1xN, Nx1; a prime side
WARP_SIZES = [((1, 1), (1, 1)), ((5, 7), (1, 13)), ((7, 5), (13, 1)), ((9, 11), (3, 7)), ((9, 11), (5, 3)), ((17, 23), (7, 9)),
              ((17, 23), (16, 16)), ((31, 37), (29, 31))]


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("src_hw,dst_hw", WARP_SIZES, ids=["%dx%d_to_%dx%d" % (a + b) for a, b in WARP_SIZES])
def test_warp_perspective_u8(monkeypatch, C, src_hw, dst_hw):
    (h, w), (dh, dw) = src_hw, dst_hw
    rng = np.random.default_rng(h * 100 + dw * 10 + C)
    src = rng.integers(0, 256, (3, h, w, C), np.uint8)
    M = np.stack([T(0.5, -0.25), np.array([[1.1, 0.05, -1.5], [-0.02, 0.9, 0.75], [1e-3, -2e-3, 1.0]]),
                  np.array([[0.7, 0.2, 2.0], [0.1, 1.3, -1.0], [0.0, 0.0, 1.0]])])
    got = run(monkeypatch, lambda fr, p, s, m: _ops().warp_perspective_u8(s, m, dh, dw),
              lambda fr, p: (IN(fr, p, src, name="src"), IN(fr, p, M, name="M")))
    for k in range(3):
        ref = cv2.warpPerspective(src[k] if C == 3 else src[k, ..., 0], M[k], (dw, dh)).reshape(dh, dw, C)
        assert np.array_equal(got[k], ref), k
        assert np.array_equal(got[k], WP.warp_perspective(src[k], M[k], (dw, dh)).reshape(dh, dw, C)), k


@pytest.mark.parametrize("h,w", [(1, 1), (1, 7), (7, 1), (5, 7), (9, 13), (16, 16), (17, 23)])
def test_gen_warp_u8_and_gray_u8(monkeypatch, h, w):
    rng = np.random.default_rng(h * 31 + w)
    img = rng.integers(0, 256, (3, h, w, 3), np.uint8)
    th = np.eye(3)[None] + rng.standard_normal((3, 3, 3)) * np.array([[0.3, 0.3, 0.5], [0.3, 0.3, 0.5], [0.2, 0.2, 0.3]])
    gray, warped, wgray = run(monkeypatch, lambda fr, p, s, t: _ops().gen_warp_u8(s, t),
                              lambda fr, p: (IN(fr, p, img, name="bgr"), IN(fr, p, th, name="theta")))
    for k in range(3):
        g = OG.gray(img[k])
        assert np.array_equal(gray[k], g) and np.array_equal(warped[k], OG.warp(img[k], th[k]))
        assert np.array_equal(wgray[k], OG.warp(g, th[k])), k
    for n in range(1, 6):                                       # numel = 1 .. 5: every residue mod 4
        px = img.reshape(-1, 3)[:n]
        got = run(monkeypatch, lambda fr, p, s: _ops().gray_u8(s), lambda fr, p: (IN(fr, p, px, name="px"),))
        assert np.array_equal(got, OG.gray(px[None])[0]), n


@pytest.mark.parametrize("sh,sw,dh,dw", [(1, 1, 1, 1), (5, 7, 1, 13), (7, 5, 13, 1), (9, 11, 5, 3), (17, 23, 7, 9), (16, 16, 33, 31)])
def test_resize_linear_u8(monkeypatch, sh, sw, dh, dw):
    src = np.random.default_rng(sh + dw).integers(0, 256, (3, sh, sw, 3), np.uint8)
    got = run(monkeypatch, lambda fr, p, s: _ops().resize_linear_u8(s, dh, dw), lambda fr, p: (IN(fr, p, src, name="src"),))
    for k in range(3):
        assert np.array_equal(got[k], cv2.resize(src[k], (dw, dh), interpolation=cv2.INTER_LINEAR)), k


@pytest.mark.parametrize("sh,sw,dh,dw", [(1, 1, 2, 3), (2, 3, 3, 5), (5, 7, 9, 13), (9, 11, 17, 23), (16, 16, 17, 33)])
def test_resize_area_up_u8(monkeypatch, sh, sw, dh, dw):
    src = np.random.default_rng(sh * 7 + dw).integers(0, 256, (3, sh, sw, 3), np.uint8)
    got = run(monkeypatch, lambda fr, p, s: _ops().resize_area_up_u8(s, dh, dw), lambda fr, p: (IN(fr, p, src, name="src"),))
    for k in range(3):
        assert np.array_equal(got[k], Z.resize_area_up_u8(src[k], dh, dw)), k


REAL_SMEM_MAX = 227 * 1024                                      # kRealPrepSmemMax: past it the source rows are read from global


REAL_GLOBAL = [(300, 4000, 17, 23), (64, 4000, 4, 190)]         # source rows per output row past shared memory


# output rows around kRealRowsPerCta = 16 on the staged path, the table-free path, and two sources whose rows per output row
# do not fit shared memory (the global-memory path; 300 x 4000 -> 17 x 23 also keeps the output rows around 16)
@pytest.mark.parametrize("FH,FW,Hh,W", [(17, 23, 15, 19), (34, 23, 16, 19), (35, 23, 17, 19), (23, 31, 1, 29), (240, 320, 142, 190),
                                         (16, 16, 16, 16)] + REAL_GLOBAL)
@pytest.mark.parametrize("mode", ["train", "test"])
def test_real_prep(monkeypatch, FH, FW, Hh, W, mode):
    from unsuperviseddeephomographyral2018_b200 import _lib
    max_rows = _ops().area_table(FH, FW, Hh, W)[1] if (FH, FW) != (Hh, W) else 0
    staged = _lib.lib.udh_real_prep_smem_bytes(max_rows, FW) <= REAL_SMEM_MAX
    assert staged == ((FH, FW, Hh, W) not in REAL_GLOBAL), (max_rows, _lib.lib.udh_real_prep_smem_bytes(max_rows, FW))
    rng = np.random.default_rng(FW * 3 + Hh)
    I, Ip = (rng.integers(0, 256, (3, FH, FW, 3)).astype(np.uint8) for _ in range(2))
    tables, _ = Z.draw_tables(rng, 3, 0.7, mode)
    outs = run(monkeypatch, lambda fr, p, a, b, t: _ops().real_prep(a, b, t, Hh, W),
               lambda fr, p: (IN(fr, p, I, name="I"), IN(fr, p, Ip, name="Ip"), IN(fr, p, tables, name="luts")))
    for t, got in enumerate(outs):
        for j in range(3):
            v = tables[j, t][(I if t % 2 == 0 else Ip)[j], np.arange(3)]
            ref = v if (FH, FW) == (Hh, W) else Z.resize_area_down_f32(v, Hh, W)
            assert np.array_equal(got[j].view(np.uint32), np.asarray(ref, np.float32).view(np.uint32)), (t, j)


# ---- ECC --------------------------------------------------------------------------------------------------------------------
# planes 2 px wide and high, and pixel counts 16 383 / 16 384 / 16 385 around the split kernel's tile
ECC_SHAPES = [(2, 40), (40, 2), (3, 5), (127, 129), (128, 128), (5, 3277)]


def _ecc_planes(B, h, w, seed):
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    rng = np.random.default_rng(seed)
    out = []
    for k in range(B):
        img = 128 + 60 * np.sin(xs / (5.0 + k) + 0.3 * k) * np.cos(ys / 7.0) + rng.normal(0, 4, (h, w))
        out.append(np.clip(img, 0, 255).astype(np.uint8))
    T0 = np.stack(out)
    I0 = np.stack([np.clip(E.warp_linear(t.astype(np.float32), np.linalg.inv(np.array(
        [[1.0, 0.003, 0.4], [-0.002, 1.0, -0.3], [0.0, 0.0, 1.0]], np.float32))), 0, 255).astype(np.uint8) for t in T0])
    return T0, I0


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("h,w", ECC_SHAPES)
def test_ecc_prep_and_both_ecc_kernels(monkeypatch, h, w, B):
    ops = _ops()
    rng = np.random.default_rng(h * w + B)
    I, Ip = (rng.integers(0, 256, (B, h, w, 3), np.uint8) for _ in range(2))
    aug = np.zeros((B, 11), np.float32)
    aug[0] = [1, 1.1, 1.3, 0.9, 1.05, 1.15, 0.85, 0.7, 1.1, 0.95, 1.0]
    for a in (aug, None):
        g1, g2 = run(monkeypatch, lambda fr, p, x, y, t: ops.ecc_prep_u8(x, y, t),
                     lambda fr, p: (IN(fr, p, I, name="I"), IN(fr, p, Ip, name="Ip"), None if a is None else IN(fr, p, a, name="aug")))
        r1, r2 = E.prep(I, Ip, a)
        assert np.array_equal(g1, r1) and np.array_equal(g2, r2)
    T0, I0 = _ecc_planes(B, h, w, h + w)
    W0 = np.tile(np.eye(3, dtype=np.float32), (B, 1, 1))
    W0[:, 0, 2] = 0.25
    for fn in (ops.find_homography_ecc, ops.find_homography_ecc_split):
        ref = [t.cpu().numpy() for t in fn(torch.from_numpy(T0).cuda(), torch.from_numpy(I0).cuda(), torch.from_numpy(W0).cuda(), 3)]
        got = run(monkeypatch, lambda fr, p, t, i, w0: fn(t, i, w0, 3),
                  lambda fr, p: (IN(fr, p, T0, name="T"), IN(fr, p, I0, name="I"), IN(fr, p, W0, name="W0")))
        BC.bit_equal(list(got), ref, fn.__name__)                # a run on plain allocations gives the same bits
        for k in range(B if min(h, w) > 3 else 0):               # (3 x 5 is too small for the oracle's stopping rule)
            o = E.ecc(T0[k], I0[k], W_init=W0[k], max_iters=3)
            assert (got[3][k], got[2][k]) == (o["status"], o["iters"]), (fn.__name__, k)


@pytest.mark.parametrize("B", [1, 3, 129])
def test_ecc_h4p_and_corr_h4p(monkeypatch, B):
    ops = _ops()
    rng = np.random.default_rng(B)
    W = np.tile(np.eye(3, dtype=np.float32), (B, 1, 1))
    W[:, :2, :2] += rng.normal(0, .02, (B, 2, 2)); W[:, :2, 2] += rng.normal(0, 10, (B, 2)); W[:, 2, :2] += rng.normal(0, 1e-4, (B, 2))
    st = np.zeros(B, np.int32)
    st[-1] = E.ECC_NOCONV
    pts1 = rng.uniform(0, 300, (B, 8)).astype(np.float32)
    gt = rng.normal(0, 8, (B, 8)).astype(np.float32)
    pred, h, fail = run(monkeypatch, lambda fr, p, w, s, a, g: ops.ecc_h4p(w, s, a, g, 45.0),
                        lambda fr, p: (IN(fr, p, W), IN(fr, p, st), IN(fr, p, pts1), IN(fr, p, gt)))
    for s in range(B):
        rp, rh, rf = E.h4p(W[s], int(st[s]), pts1[s], gt[s])
        assert np.array_equal(pred[s], rp) and int(fail[s]) == rf and float(h[s]) == pytest.approx(rh, rel=1e-6), s
    c1 = rng.uniform(40, 600, (B, 8))
    g16 = np.concatenate([c1, c1 + rng.normal(0, 8, (B, 8))], 1).astype(np.float32)
    pred, h, fail = run(monkeypatch, lambda fr, p, w, s, g: ops.ecc_corr_h4p(w, s, g),
                        lambda fr, p: (IN(fr, p, W), IN(fr, p, st), IN(fr, p, g16)))
    rp, rh, rf = R.corr_h4p(W, st, g16)
    assert np.array_equal(fail, rf) and np.array_equal(h.view(np.uint64), rh.view(np.uint64))
    assert np.array_equal(pred.view(np.uint32), np.asarray(rp, np.float32).view(np.uint32))


# ---- mosaic blends ----------------------------------------------------------------------------------------------------------
def mosaic_case(name):
    """(frames uint8 RGB, M, (Hc, Wc)) with the edges of the blends' tiles: canvas sides 1, 31, 33 (16 x 64 feather
    tiles, 32 x 8 multi-band tiles), a frame 1 px wide, a frame whose ROI misses the canvas, and a small sweep."""
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "row":                                            # canvas 1 x 33
        sizes, M, canvas = [(3, 20), (4, 25)], [T(-0.5, -1), T(10.25, -2)], (1, 33)
    elif name == "column":                                       # canvas 31 x 1, a frame 1 px wide
        sizes, M, canvas = [(20, 3), (25, 1)], [T(-1, -0.5), T(0, 8)], (31, 1)
    elif name == "ragged":                                       # canvas 33 x 31, a frame that misses it, a 1-px-wide frame
        sizes, M, canvas = [(20, 18), (22, 16), (9, 1), (6, 6)], [T(-1.5, 2.25), T(14, 9.5), T(7, 3), T(100, 100)], (33, 31)
    elif name == "wide":                                         # canvas 31 x 65: one feather tile plus one column
        sizes, M, canvas = [(25, 40), (28, 36), (1, 30)], [T(0.5, 1), T(27, 2.5), T(5, 15)], (31, 65)
    elif name == "sweep":
        _, frames, _, H = SW.sweep(3, 40, 56, seed=5)
        import test_seam_logic as SL
        return SL._chain(frames, H)
    frames = [rng.integers(0, 256, (h, w, 3), np.uint8) for h, w in sizes]
    return frames, np.stack(M), canvas


MOSAIC_CASES = ["row", "column", "ragged", "wide", "sweep"]


def _frames_in(frames):
    return lambda fr, p: tuple(IN(fr, p, f, name="frame%d" % k) for k, f in enumerate(frames))


def _extras(frames, M, Hc, Wc, variant):
    """Host arrays of one blend variant -> (kwargs builder on framed copies, oracle feather (px), oracle multiband (bands))."""
    ops = _ops()
    if variant == "plain":
        return (lambda fr, p: {}, lambda f: OM.blend(frames, M, Hc, Wc, f), lambda b: MB.blend(frames, M, Hc, Wc, b))
    if variant == "gains":
        g = np.linspace(0.8, 1.25, len(frames) * 3).reshape(-1, 3)
        return (lambda fr, p: dict(gains=g), lambda f: EX.feather(frames, M, Hc, Wc, f, g), lambda b: EX.multiband(frames, M, Hc, Wc, b, g))
    if variant == "masks":
        sm = ops.mosaic_seam_masks([torch.from_numpy(f).cuda() for f in frames], M, Hc, Wc)
        blend = [b.cpu().numpy() for b in sm["blend"]]
        full = [None] * len(frames)
        for q, k in enumerate(sm["take"]):
            full[k] = blend[q]

        def kw(fr, p):
            return dict(masks=[None if b is None else IN(fr, p, b, name="mask%d" % k) for k, b in enumerate(full)])
        return kw, lambda f: SM.feather(frames, M, Hc, Wc, f), lambda b: SM.multiband(frames, M, Hc, Wc, b)
    maps = ops.mosaic_exposure_gain_maps([torch.from_numpy(f).cuda() for f in frames], M, Hc, Wc, "channels", 1, 16)
    host = [None if m is None else m.cpu().numpy() for m in maps]

    def kw(fr, p):
        return dict(gain_maps=[None if m is None else IN(fr, p, m, name="map%d" % k) for k, m in enumerate(host)])
    return kw, lambda f: XB.feather(frames, M, Hc, Wc, f, host), lambda b: XB.multiband(frames, M, Hc, Wc, b, host)


@pytest.mark.parametrize("variant", ["plain", "gains", "masks", "gain_maps"])
@pytest.mark.parametrize("name", MOSAIC_CASES)
def test_mosaic_blend_u8(monkeypatch, name, variant):
    ops = _ops()
    frames, M, (Hc, Wc) = mosaic_case(name)
    kw, ref_feather, _ = _extras(frames, M, Hc, Wc, variant)
    for feather in (0, 1):
        got = run(monkeypatch, lambda fr, p, *fs: ops.mosaic_blend_u8(list(fs), M, Hc, Wc, feather, **kw(fr, p)), _frames_in(frames))
        ref = ref_feather(feather)
        assert np.array_equal(got[1], ref[1]) and np.array_equal(got[0], ref[0]), feather


@pytest.mark.parametrize("variant", ["plain", "gains", "masks", "gain_maps"])
@pytest.mark.parametrize("name", MOSAIC_CASES)
def test_mosaic_multiband_u8(monkeypatch, name, variant):
    ops = _ops()
    frames, M, (Hc, Wc) = mosaic_case(name)
    kw, _, ref_mb = _extras(frames, M, Hc, Wc, variant)
    top = max(1, int(np.log2(max(Hc, Wc))) + 1)                  # every band count up to where a level is 1 px
    for bands in range(0, top + 1):
        got = run(monkeypatch, lambda fr, p, *fs: ops.mosaic_multiband_u8(list(fs), M, Hc, Wc, bands, **kw(fr, p)), _frames_in(frames))
        ref = ref_mb(bands)
        assert np.array_equal(got[1], ref[1]) and np.array_equal(got[0], ref[0]), bands


def seam_case(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    if name.startswith("w"):                                     # canvas widths around the 1 024-px row chunk
        Wc = int(name[1:])
        sizes, M, canvas = [(15, 600), (17, 560)], [T(0, 0.5), T(Wc - 560, 0)], (17, Wc)
    elif name.startswith("h"):                                   # heights around 16 row segments
        Hc = int(name[1:])
        sizes, M, canvas = [(Hc, 30), (Hc - 1, 25)], [T(0, 0), T(12.5, 1)], (Hc, 40)
    else:                                                        # frame 1 inside frame 0, frame 2 inside frame 1
        sizes, M, canvas = [(40, 50), (20, 24), (6, 6)], [T(1, 1), T(13, 10), T(21, 16)], (42, 52)
    return [rng.integers(0, 256, (h, w, 3), np.uint8) for h, w in sizes], np.stack(M), canvas


@pytest.mark.parametrize("name", ["w1023", "w1024", "w1025", "h15", "h16", "h17", "h33", "contained"])
def test_mosaic_seam_masks(monkeypatch, name):
    ops = _ops()
    frames, M, (Hc, Wc) = seam_case(name)
    got = run(monkeypatch, lambda fr, p, *fs: {k: v for k, v in ops.mosaic_seam_masks(list(fs), M, Hc, Wc).items() if k != "rois"},
              _frames_in(frames))
    take, _, masks, tls = SM.fed(frames, M, Hc, Wc)
    seams = SM.cv2_seams(masks, tls)
    assert list(got["take"]) == take
    for k, (s, b, rs, rb) in enumerate(zip(got["seam"], got["blend"], seams, SM.blend_masks(seams, masks))):
        assert np.array_equal(s, rs) and np.array_equal(b, rb), k


# ---- exposure ---------------------------------------------------------------------------------------------------------------
def exposure_case(name):
    if name == "one":                                            # n = 1
        rng = np.random.default_rng(1)
        return [rng.integers(0, 256, (30, 60, 3), np.uint8)], T(1, 1)[None], (31, 63)
    if name == "grid":                                           # canvases around the 32 x 64 statistics tile
        rng = np.random.default_rng(2)
        sizes, M, canvas = [(33, 65), (31, 63), (32, 64)], [T(0, 0), T(20.5, 1.25), T(-3, 15)], (45, 83)
        return [rng.integers(0, 256, (h, w, 3), np.uint8) for h, w in sizes], np.stack(M), canvas
    return mosaic_case(name)


def _ref_stats(frames, M, Hc, Wc, hist):
    take, imgs, masks, tls = EX.fed(frames, M, Hc, Wc)
    cur = list(imgs)
    for g in hist:
        cur = [EX.apply(img, gk) for img, gk in zip(cur, g)]
    return {(p["i"], p["j"]): p for p in EX.pair_stats(cur, masks, tls, "exact")}


@pytest.mark.parametrize("name", ["one", "grid", "ragged", "sweep"])
def test_exposure_stats_across_feeds(monkeypatch, name):
    ops = _ops()
    frames, M, (Hc, Wc) = exposure_case(name)
    m = len(EX.fed(frames, M, Hc, Wc)[0])
    hist = np.random.default_rng(m).uniform(0.7, 1.4, (2, m, 3))

    def call(fr, p, *fs):
        st = ops._ExposureStats(list(fs), M, Hc, Wc)
        out = []
        for t in (0, 1, 2, 0):                                   # the last call repeats the first on a re-poisoned workspace
            out.append(st(hist[:t] if t else None).copy())
            fr.poison(st.ws, p ^ 0xFF)
            fr.poison(st.out, p ^ 0xFF)
        return out, st.i, st.j

    (raws, i, j) = run(monkeypatch, call, _frames_in(frames))
    BC.bit_equal(raws[0], raws[3])
    for t in range(3):
        ref = _ref_stats(frames, M, Hc, Wc, hist[:t])
        for q, key in enumerate(zip(i.tolist(), j.tolist())):
            r = raws[t][q]
            assert r[0] == ref[key]["count"] and np.array_equal(r[1:7].astype(np.int64).reshape(2, 3), ref[key]["sums"]), (t, key)
            assert [ops.exposure_norm_sum(*r[7:10]), ops.exposure_norm_sum(*r[10:13])] == list(ref[key]["norms"]), (t, key)


@pytest.mark.parametrize("block", [16, 32, 48])
@pytest.mark.parametrize("name", ["one", "grid", "sweep"])
def test_exposure_block_stats_solve_and_maps(monkeypatch, name, block):
    ops = _ops()
    frames, M, (Hc, Wc) = exposure_case(name)
    take, imgs, masks, tls = EX.fed(frames, M, Hc, Wc)
    bi, bm, bt, _ = XB.blocks(imgs, masks, tls, block, block)
    hist = np.random.default_rng(block).uniform(0.7, 1.4, (2, len(bi), 3))

    def call(fr, p, *fs):
        st = ops._ExposureBlockStats(list(fs), M, Hc, Wc, block)
        # each history prefix framed on its own, so a read past the t rows the kernel is given hits the poison
        h_d = [None] + [IN(fr, p, hist[:t], name="history%d" % t) for t in (1, 2)]
        out = []
        for t in (0, 1, 2, 0):
            out.append(st(h_d[t]).copy())
            fr.poison(st.ws, p ^ 0xFF)
            fr.poison(st.out, p ^ 0xFF)
        return out, st.cells["a"], st.cells["b"]

    raws, a, b = run(monkeypatch, call, _frames_in(frames))
    BC.bit_equal(raws[0], raws[3])
    for t in range(3):
        cur = [np.asarray(x) for x in bi]
        for g in hist[:t]:
            cur = [EX.apply(img, gk) for img, gk in zip(cur, g)]
        ref = {(q["i"], q["j"]): q for q in EX.pair_stats(cur, bm, bt, "exact")}
        for q, key in enumerate(zip(a.tolist(), b.tolist())):
            assert raws[t][q][0] == ref[key]["count"], (t, key)
            assert np.array_equal(raws[t][q][1:7].astype(np.int64).reshape(2, 3), ref[key]["sums"]), (t, key)
    # the solver (one CTA, fixed reductions) and the map filter repeat exactly: bit for bit across the poisons
    got = run(monkeypatch, lambda fr, p, *fs: ops.mosaic_exposure_block_gains(list(fs), M, Hc, Wc, "channels", 2, block)["gains"],
              _frames_in(frames))
    ref_g = XB.restate(imgs, masks, tls, "channels", 2, block)[1]
    assert np.abs(got - ref_g).max() <= 1e-12                     # the bound of test_gpu_exposure_blocks
    maps = run(monkeypatch, lambda fr, p, *fs: [m for m in ops.mosaic_exposure_gain_maps(list(fs), M, Hc, Wc, "gain", 1, block)
                                                 if m is not None], _frames_in(frames))
    ref_maps = XB.restate(imgs, masks, tls, "gain", 1, block)[0]
    assert len(maps) == len(ref_maps)
    for mp, rm in zip(maps, ref_maps):
        assert rel_l2(mp, rm) <= 1e-6


# ---- decoders and the encoder ---------------------------------------------------------------------------------------------
JPEG_SIZES = J.SIZES + [(7, 9), (8, 8), (9, 17), (15, 15), (16, 16), (17, 17)]


def _jpeg_parallel(mode):
    from unsuperviseddeephomographyral2018_b200 import _lib

    @contextlib.contextmanager
    def ctx():
        _lib.check(_lib.lib.udh_debug_jpeg_set_parallel(mode))
        try:
            yield
        finally:
            _lib.check(_lib.lib.udh_debug_jpeg_set_parallel(-1))
    return ctx()


@pytest.mark.parametrize("path", [0, 1], ids=["serial", "parallel"])
@pytest.mark.parametrize("h,w", JPEG_SIZES)
def test_jpeg_decode(monkeypatch, h, w, path):
    ops = _ops()
    files = [b for _, b in J.corpus(h, w)]
    bad = len(files) // 2 if h * w > 1 else None                 # a file whose entropy data is cut short among good ones
    blobs = list(files)
    if bad is not None:
        sos = files[bad].rfind(b"\xff\xda")
        blobs.insert(bad, files[bad][:len(files[bad]) - max(2, (len(files[bad]) - sos) // 2)])

    def call(fr, p):
        plan = ops.JpegPlan(blobs, h, w)
        outs = []
        for _ in range(2):                       # the plan decoded twice; each decode takes a fresh (poisoned) workspace
            out, status = plan.decode()
            st = status.cpu().numpy()
            keep = [k for k in range(len(blobs)) if k != bad]
            outs.append((out[keep].cpu().numpy(), st))
        return outs

    with _jpeg_parallel(path):
        outs = run(monkeypatch, call)
    BC.bit_equal(outs[0], outs[1])
    got, st = outs[0]
    if bad is not None:
        assert st[bad] != 0
        st = np.delete(st, bad)
    assert (st == 0).all()
    for k, blob in enumerate(files):
        ref = cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)[..., ::-1]
        assert np.array_equal(got[k], ref), k


@pytest.mark.parametrize("h,w", PNG.SIZES + [(7, 9), (8, 8), (9, 17), (16, 16)])
def test_png_decode(monkeypatch, h, w):
    ops = _ops()
    files = [b for _, b in PNG.corpus(h, w)]
    got, st = run(monkeypatch, lambda fr, p: ops.decode_png(files, h, w))
    assert (st == 0).all()
    for k, blob in enumerate(files):
        assert np.array_equal(got[k], cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)), k


@pytest.mark.parametrize("channels", [3, 1])
@pytest.mark.parametrize("h,w", [(1, 1), (7, 9), (8, 8), (9, 17), (15, 15), (16, 16), (17, 17), (17, 23)])
def test_jpeg_encode(monkeypatch, h, w, channels):
    ops = _ops()
    imgs = np.stack([JE.image(k, h, w, channels, seed=3) for k in JE.KINDS[:3]])

    def call(fr, p, x):
        out, nb, st = ops.encode_jpeg_device(x, 95)
        n = nb.cpu().numpy()
        return [out[k, :int(n[k])] for k in range(len(n))], st

    files, st = run(monkeypatch, call, lambda fr, p: (IN(fr, p, imgs, name="imgs"),))
    assert (st == 0).all()
    for k in range(len(imgs)):
        ok, buf = cv2.imencode(".jpg", imgs[k], [cv2.IMWRITE_JPEG_QUALITY, 95])
        assert files[k].tobytes() == buf.tobytes(), k


# ---- report drawing -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("h,w", [(1, 1), (7, 9), (17, 23)])
def test_draw_report_u8(monkeypatch, B, h, w):
    ops = _ops()
    rng = np.random.default_rng(B * 100 + h)
    I, Ip = (rng.integers(0, 256, (B, h, w, 3), np.uint8) for _ in range(2))
    verts = D.vertex_cases(rng, B, h, w)
    verts[0, :4] = [[-50, -50], [3 * w, -7], [3 * w, 2 * h], [-9, 2 * h]]          # vertices off the image
    got = run(monkeypatch, lambda fr, p, a, b, v: ops.draw_report_u8(a, b, None, v, True),
              lambda fr, p: (IN(fr, p, I, name="I"), IN(fr, p, Ip, name="Ip"), IN(fr, p, verts, name="verts")))
    for k in range(B):
        ref = D.cv2_draw_report(D.host_denorm(Ip[k], None, 1), D.host_denorm(I[k], None, 0), verts[k])
        assert np.array_equal(got[k], ref), k


# ---- the photometric path ---------------------------------------------------------------------------------------------------
def _photo_inputs(B, C, pw, ph, Hh, W, seed):
    rng = np.random.default_rng(seed)
    I = rng.uniform(-1, 1, (B, Hh, W, C)).astype(np.float32)
    ox = np.where(np.arange(B) % 3 == 0, 0, np.where(np.arange(B) % 3 == 1, W - pw, rng.integers(0, W - pw + 1, B)))
    oy = np.where(np.arange(B) % 2 == 0, 0, Hh - ph)                  # windows at the image's corners
    ys, xs = np.mgrid[0:ph, 0:pw]
    idx = ((oy[:, None, None] + ys) * W + ox[:, None, None] + xs).reshape(B, -1).astype(np.int32)
    H = np.tile(np.eye(3, dtype=np.float32), (B, 1, 1))
    H[:, :2, 2] = rng.normal(0, 1.5, (B, 2)) + np.stack([ox, oy], 1)
    H[:, :2, :2] += rng.normal(0, 0.01, (B, 2, 2)).astype(np.float32)
    I2 = rng.uniform(-1, 1, (B, ph, pw, 1)).astype(np.float32)
    return I, H, I2, idx


@pytest.mark.parametrize("B", [1, 3, 129])
@pytest.mark.parametrize("C,pw,ph,Hh,W", [(1, 12, 11, 17, 23), (3, 16, 16, 16, 16), (1, 128, 128, 240, 320)])
def test_photometric_path(monkeypatch, B, C, pw, ph, Hh, W):
    ops = _ops()
    from unsuperviseddeephomographyral2018_b200 import _lib
    if B == 129 and pw == 128:
        B = 64                                                    # the full grid at the engine's patch; keeps the run short
    I, H, I2, idx = _photo_inputs(B, C, pw, ph, Hh, W, B * 7 + pw)

    def call(fr, p, i, hm, i2, ix):
        pred, sums = ops.warp_loss_forward(i, hm, i2, ix, pw, ph)
        losses = ops.photo_losses(pred, i2, sums.clone(), pw, ph, B)
        dpred = ops.ssim_backward(pred, i2, pw, ph)
        dH = [ops.warp_loss_backward(i, hm, i2, ix, pw, ph, lt, sums, 1.0) for lt in (_lib.LOSS_L1, _lib.LOSS_REC, _lib.LOSS_L1_SMOOTH)]
        dH.append(ops.warp_loss_backward(i, hm, i2, ix, pw, ph, _lib.LOSS_CUSTOM, sums, 1.0, dpred=dpred))
        return pred, dpred, sums[:6], losses[:5], dH

    inputs = lambda fr, p: (IN(fr, p, I, name="I"), IN(fr, p, H, name="H"), IN(fr, p, I2, name="I2"), IN(fr, p, idx, name="idx"))
    got = run(monkeypatch, call, inputs, same=close(1e-4))         # dH: float atomics over the window's pixels
    plain = BC.to_host(call(None, None, *(torch.from_numpy(x).cuda() for x in (I, H, I2, idx))))
    BC.bit_equal(got[:2], plain[:2])                               # pred and the SSIM gradient are deterministic
    close(1e-4)(got[2:], plain[2:])


@pytest.mark.parametrize("B", [1, 3, 129])
def test_transformer_dlt_and_h4p_loss(monkeypatch, B):
    ops = _ops()
    rng = np.random.default_rng(B)
    U = rng.uniform(-1, 1, (B, 17, 23, 3)).astype(np.float32)
    th = (np.eye(3)[None] + rng.normal(0, 0.05, (B, 3, 3))).astype(np.float32)
    pts1 = np.tile(np.array([0, 0, 127, 0, 0, 127, 127, 127], np.float32), (B, 1)) + rng.uniform(0, 50, (B, 8)).astype(np.float32)
    h4p = rng.normal(0, 10, (B, 8)).astype(np.float32)
    dH = rng.normal(0, 1, (B, 3, 3)).astype(np.float32)
    gt = rng.normal(0, 10, (B, 8)).astype(np.float32)

    def call(fr, p, u, t, a, h, d, g):
        out = [ops.transformer(u, t, (13, 11))[0]]
        Hm = ops.dlt_forward(a, h)
        out += [Hm, ops.dlt_backward(a, h, Hm, d)]
        m, per, dp = ops.h4p_loss(h, g, want_grad=True, want_per_sample=True)
        return out + [per, dp, m]

    inputs = lambda fr, p: tuple(IN(fr, p, x) for x in (U, th, pts1, h4p, dH, gt))
    got = run(monkeypatch, call, inputs, same=close(1e-6))
    plain = BC.to_host(call(None, None, *(torch.from_numpy(x).cuda() for x in (U, th, pts1, h4p, dH, gt))))
    BC.bit_equal(got[:5], plain[:5])
    close(1e-6)(got[5:], plain[5:])


@pytest.mark.parametrize("B", [1, 3, 129])
def test_synthetic_batch_kernels(monkeypatch, B):
    """udh_synth_scene_u8, udh_warp_image_u8 and udh_prep_inputs_u8_ex (synthetic.make_batch_fast) with augmentation."""
    from unsuperviseddeephomographyral2018_b200 import synthetic
    keys = ("I_u8", "I_prime_u8", "pts1", "gt", "I", "I_prime", "I_aug", "I_aug_rgb", "patch_indices")

    def call(fr, p):
        b = synthetic.make_batch_fast(B, seed=7, do_augment=1.0, want_rgb=True)
        return {k: b[k] for k in keys if b.get(k) is not None}

    got = run(monkeypatch, call, mods=[_ops(), synthetic])
    plain = BC.to_host(call(None, None))
    BC.bit_equal(got, plain)


# ---- the CNN engine's workspace --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 70, 128])
@pytest.mark.parametrize("loss", ["h_loss", "l1_loss"])
@pytest.mark.parametrize("numeric", ["fp32", "bf16", "bf16x3"])
def test_engine_workspace_poisoned_before_init(numeric, loss, B):
    from unsuperviseddeephomographyral2018_b200 import _lib, engine, ops, synthetic
    lib = _lib.lib
    engs = []
    for poisoned in (True, False):
        e = engine.HomographyEngine(B, numeric=numeric, seed=3, loss_type=loss)
        if poisoned:                                   # NaN wherever the initialisation and the step write nothing
            e.ws.fill_(0xFF)
            _lib.check(lib.udh_cnn_workspace_init(e._p(e.ws), e.ws_bytes, e.B, e.Pz, e.numeric, ops._stream()), "workspace_init")
            e._mirror_current = False
        engs.append(e)
    batches = [synthetic.make_batch_fast(B, seed=100 + k) for k in range(4)]
    keys = ("pred_h4p", "photo_losses", "h4p_metrics", "batch_h_loss")
    state = ("params", "grads", "adam_m", "adam_v")
    # bf16 / bf16x3 with h_loss step bit for bit run to run.  fp32's conv weight gradients and every mode's photometric dH
    # accumulate with atomics, so two untouched engines drift apart over steps as far as this pair does (rel L2 of m and v
    # ~1e-2 after three steps, measured both ways on one H100): there the poisoned engine starts every step from the
    # untouched one's state (its workspace kept), and each step's outputs are held to that step's atomics alone.
    exact = numeric != "fp32" and loss == "h_loss"
    res = [[], []]
    for k in range(4):
        if not exact:
            for n in state:
                getattr(engs[0], n).copy_(getattr(engs[1], n))
        for e, r in zip(engs, res):
            out = e.train_step(batches[k]) if k < 3 else e.eval_step(batches[k])
            torch.cuda.synchronize()
            r.append({n: out[n].detach().cpu().numpy().copy() for n in keys if out.get(n) is not None})
            r[-1].update({n: getattr(e, n).cpu().numpy().copy() for n in state})
    for step in res[0]:
        for n, v in step.items():
            assert np.isfinite(v).all(), (numeric, n)
    if exact:
        BC.bit_equal(res[0], res[1])
        print("%s %s B=%d: 3 steps and an eval bit-identical to an untouched engine" % (numeric, loss, B))
        return
    # each step from a shared state: the forward is deterministic, so pred_h4p (three steps and the eval) is bit for bit;
    # the losses and metrics, and per tensor the gradients and Adam's m and v, are within test_gpu_train_loop's 1e-4
    # rel-L2 envelope; the parameters as a whole (a near-zero bias moved by Adam's normalised step can exceed it alone).
    # Single-pass bf16 rounds the backward's operands to 8 bits, which turns the dH atomics' ~1e-6 into whole-ulp flips:
    # two untouched engines differ by up to 1.7e-3 per tensor there (measured on one H100), so its envelope is 1e-2.
    tol = 1e-2 if numeric == "bf16" else 1e-4
    specs = list(engs[1].specs.values())
    worst = 0.0
    for k, (a, b) in enumerate(zip(res[0], res[1])):
        BC.bit_equal(a["pred_h4p"], b["pred_h4p"], "pred_h4p at step %d" % k)
        for n in keys[1:]:
            if n in a:
                worst = max(worst, rel_l2(a[n], b[n]))
                assert rel_l2(a[n], b[n]) < tol, (k, n, rel_l2(a[n], b[n]))
        for n in ("grads", "adam_m", "adam_v"):
            for sp in specs:
                r = rel_l2(a[n][sp.offset:sp.offset + sp.size], b[n][sp.offset:sp.offset + sp.size])
                worst = max(worst, r)
                assert r < tol, (k, n, sp.name, r)
        r = rel_l2(a["params"], b["params"])
        worst = max(worst, r)
        assert r < tol, (k, "params", r)
    print("%s %s B=%d: pred_h4p bit-identical at every step and the eval, worst rel L2 %.2e, all finite" % (numeric, loss, B, worst))
