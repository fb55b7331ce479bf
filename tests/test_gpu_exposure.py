"""GPU tests of the mosaic's exposure compensation: udh_mosaic_exposure_stats_u8's pair statistics against the NumPy
restatement (oracle/exposure.py) exactly, the gains against cv2's compensators, both compensated blends against their
oracles byte for byte, order and run independence, unit gains against the uncompensated kernels, a 12 MP sweep with known
exposures, and mosaic_images.py --compensate end to end."""
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
import test_gpu_mosaic as GM  # noqa: E402
from oracle import exposure as EX  # noqa: E402

pytestmark = pytest.mark.gpu


def _cuda(frames):
    return [torch.from_numpy(np.ascontiguousarray(f)).cuda() for f in frames]


def stacked_case(n=20, seed=3):
    """n frames of 24 x 30 within a few pixels of each other, each with its own exposure: more than 8 frames meet every
    tile, so the kernel takes its frames in several chunks."""
    rng = np.random.default_rng(seed)
    frames = [np.clip(rng.integers(0, 200, (24, 30, 3)) * rng.uniform(0.7, 1.3), 0, 255).astype(np.uint8) for _ in range(n)]
    M = np.stack([GM.T(2 + (k % 5), 3 + (k % 3)) for k in range(n)])
    return frames, M, (33, 41)


def sweep_case(n=4, h=240, w=320, seed=9, exposures=None):
    from unsuperviseddeephomographyral2018_b200 import mosaic
    _, frames, _, H = SW.sweep(n, h, w, seed=seed)
    if exposures is not None:
        frames = [EX.apply(f, 0.7 * e) for f, e in zip(frames, exposures)]
    G, ref = mosaic.chain_to_reference(H)
    M, (Hc, Wc), kept = mosaic.canvas([f.shape[:2] for f in frames], G, ref)
    assert kept.all()
    return frames, M, (Hc, Wc)


def case(name):
    if name == "stacked":
        return stacked_case()
    if name == "stacked40":                                   # every tile's frames are listed by two warps
        return stacked_case(40, seed=4)
    if name == "stacked300":                                  # ... and in two rounds of 256
        return stacked_case(300, seed=5)
    if name == "sweep":
        return sweep_case(exposures=(0.8, 1.0, 1.25, 0.9))
    frames, M, canvas = GM._case(name, 3, np.random.default_rng(17))
    frames = [EX.apply(f, 0.5 + 0.2 * k) for k, f in enumerate(frames)]
    return frames, M, canvas


CASES = ["two", "seven", "stacked", "stacked40", "sweep"]


# ---- statistics ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("feeds", [0, 2])
@pytest.mark.parametrize("name", CASES + ["stacked300"])
def test_stats_equal_the_restatement(name, feeds):
    """Counts and channel sums exactly; the norm sums bit for bit with math.fsum of the same norms.  feeds: the statistics
    of images compensated by that many earlier feeds' gains first."""
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case(name)
    take, imgs, masks, tls = EX.fed(frames, M, Hc, Wc)
    rng = np.random.default_rng(feeds)
    hist = rng.uniform(0.7, 1.4, (feeds, len(take), 3)) if feeds else None
    got = ops.mosaic_exposure_stats(_cuda(frames), M, Hc, Wc, history=hist)
    assert got["take"] == take
    for t in range(feeds):
        imgs = [EX.apply(img, hist[t, k]) for k, img in enumerate(imgs)]
    ref = EX.pair_stats(imgs, masks, tls, "exact")
    assert [(p["i"], p["j"]) for p in ref] == list(zip(got["i"], got["j"]))
    assert np.array_equal(got["count"], [p["count"] for p in ref])
    assert np.array_equal(got["sums"], np.stack([p["sums"] for p in ref]))
    assert np.array_equal(got["norms"], np.stack([p["norms"] for p in ref]))
    assert (got["count"][got["i"] != got["j"]] > 0).any()


@pytest.mark.parametrize("name", ["seven", "stacked40"])
def test_stats_do_not_depend_on_order_or_run(name):
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case(name)
    a = ops.mosaic_exposure_stats(_cuda(frames), M, Hc, Wc)
    b = ops.mosaic_exposure_stats(_cuda(frames), M, Hc, Wc)
    assert np.array_equal(a["raw"], b["raw"])
    perm = [4, 1, 6, 0, 3, 5, 2] if name == "seven" else list(np.random.default_rng(1).permutation(len(frames)))
    c = ops.mosaic_exposure_stats(_cuda([frames[k] for k in perm]), M[perm], Hc, Wc)

    def by_frames(st, ids):
        out = {}
        for i, j, r in zip(st["i"], st["j"], st["raw"]):
            fi, fj = ids[st["take"][i]], ids[st["take"][j]]
            if fi > fj:                                       # the pair's frames swap roles
                fi, fj, r = fj, fi, np.concatenate([r[:1], r[4:7], r[1:4], r[10:13], r[7:10]])
            out[(fi, fj)] = r
        return out

    da, dc = by_frames(a, list(range(len(frames)))), by_frames(c, perm)
    assert sorted(da) == sorted(dc) and all(np.array_equal(da[k], dc[k]) for k in da)
    # the gains: the same bits run to run; in another frame order the host's LU solve meets its rows in another order, so
    # (as in cv2) they agree to rounding
    g1 = ops.mosaic_exposure_gains(_cuda(frames), M, Hc, Wc, "gain", 2)
    assert np.array_equal(g1, ops.mosaic_exposure_gains(_cuda(frames), M, Hc, Wc, "gain", 2))
    g2 = ops.mosaic_exposure_gains(_cuda([frames[k] for k in perm]), M[perm], Hc, Wc, "gain", 2)
    assert np.abs(g1[perm] / g2 - 1).max() < 1e-13


# ---- gains -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("feeds", [1, 2, 3])
@pytest.mark.parametrize("name", CASES + ["stacked300"])
def test_channels_gains_equal_cv2_bit_for_bit(name, feeds):
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case(name)
    got = ops.mosaic_exposure_gains(_cuda(frames), M, Hc, Wc, "channels", feeds)
    ref = EX.gains(frames, M, Hc, Wc, "channels", feeds)
    assert np.array_equal(got, ref)
    assert (got != 1.0).any()


@pytest.mark.parametrize("feeds", [1, 2])
@pytest.mark.parametrize("name", CASES)
def test_gain_mode_equals_the_exact_restatement(name, feeds):
    """The kernel's exact sums give the restatement's gains with exact sums bit for bit, and cv2's to its summation error."""
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case(name)
    got = ops.mosaic_exposure_gains(_cuda(frames), M, Hc, Wc, "gain", feeds)
    take, imgs, masks, tls = EX.fed(frames, M, Hc, Wc)
    ref = np.ones_like(got)
    ref[take] = EX.restate(imgs, masks, tls, "gain", feeds, "exact")[0]
    assert np.array_equal(got, ref)
    cv = EX.gains(frames, M, Hc, Wc, "gain", feeds)
    assert np.abs(got / cv - 1).max() < 1e-12


# ---- the compensated blends --------------------------------------------------------------------------------------------------
def _gains_for(frames, seed):
    rng = np.random.default_rng(seed)
    g = rng.uniform(0.6, 1.6, (len(frames), 3))
    g[0] = (1.5, 0.5, 1.0)                                     # ties on every odd value
    return g


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("name", ["one", "two", "seven"])
def test_feather_blend_with_gains_equals_the_oracle(name, C):
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = GM._case(name, C, np.random.default_rng(C))
    g = _gains_for(frames, C)
    out, mask = ops.mosaic_blend_u8(_cuda(frames), M, Hc, Wc, 64, gains=g)
    ref, ref_mask = EX.feather(frames, M, Hc, Wc, 64, g)
    assert np.array_equal(mask.cpu().numpy(), ref_mask) and np.array_equal(out.cpu().numpy(), ref)
    if C == 3:                                                 # one gain per frame is the same as [n,3] of it
        o2, _ = ops.mosaic_blend_u8(_cuda(frames), M, Hc, Wc, 64, gains=g[:, 0])
        ref2, _ = EX.feather(frames, M, Hc, Wc, 64, np.repeat(g[:, :1], 3, 1))
        assert np.array_equal(o2.cpu().numpy(), ref2)


@pytest.mark.parametrize("name", ["one", "two", "seven", "stacked"])
def test_multiband_with_gains_equals_the_oracle(name):
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case(name) if name == "stacked" else GM._case(name, 3, np.random.default_rng(5))
    g = _gains_for(frames, 5)
    out, mask = ops.mosaic_multiband_u8(_cuda(frames), M, Hc, Wc, 5, gains=g)
    ref, ref_mask = EX.multiband(frames, M, Hc, Wc, 5, g)
    assert np.array_equal(mask.cpu().numpy(), ref_mask) and np.array_equal(out.cpu().numpy(), ref)


@pytest.mark.parametrize("blend", ["feather", "multiband"])
def test_unit_gains_give_the_uncompensated_bytes(blend):
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = GM._case("seven", 3, np.random.default_rng(2))
    one = np.ones((len(frames), 3))
    if blend == "feather":
        a = ops.mosaic_blend_u8(_cuda(frames), M, Hc, Wc, 64)
        b = ops.mosaic_blend_u8(_cuda(frames), M, Hc, Wc, 64, gains=one)
    else:
        a = ops.mosaic_multiband_u8(_cuda(frames), M, Hc, Wc, 5)
        b = ops.mosaic_multiband_u8(_cuda(frames), M, Hc, Wc, 5, gains=one)
    assert all(np.array_equal(x.cpu().numpy(), y.cpu().numpy()) for x, y in zip(a, b))


# ---- end to end against cv2 ----------------------------------------------------------------------------------------------------
def _near_ties(frames, M, Hc, Wc, g_a, g_b):
    """Fed pixels v whose v g lies within v |g_a - g_b| of a tie (x.5): the only places where apply can round two gains
    that differ by that much apart."""
    take, imgs, _, _ = EX.fed(frames, M, Hc, Wc)
    n = 0
    for img, k in zip(imgs, take):
        v = img.astype(np.float64)
        x = v * g_a[k]
        n += int((np.abs(x - np.floor(x) - 0.5) <= v * np.abs(g_a[k] - g_b[k]) + 1e-9).sum())
    return n


@pytest.mark.parametrize("mode", ["channels", "gain"])
@pytest.mark.parametrize("name", ["seven", "sweep"])
def test_end_to_end_against_cv2(name, mode):
    """cv2's compensator, then the existing oracles, against the GPU gains and compensated blends.  Channels: byte for
    byte.  Gain: the gains differ by cv2's summation error, so a byte could differ only where v g is that close to a tie;
    there are no such pixels in these cases, and the bytes are equal."""
    from unsuperviseddeephomographyral2018_b200 import ops
    frames, M, (Hc, Wc) = case(name)
    g = ops.mosaic_exposure_gains(_cuda(frames), M, Hc, Wc, mode, 1)
    cv = EX.gains(frames, M, Hc, Wc, mode, 1)
    if mode == "channels":
        assert np.array_equal(g, cv)
    else:
        assert _near_ties(frames, M, Hc, Wc, cv, g) == 0
    out, mask = ops.mosaic_multiband_u8(_cuda(frames), M, Hc, Wc, 5, gains=g)
    ref, ref_mask = EX.multiband(frames, M, Hc, Wc, 5, cv)
    assert np.array_equal(out.cpu().numpy(), ref) and np.array_equal(mask.cpu().numpy(), ref_mask)
    out, mask = ops.mosaic_blend_u8(_cuda(frames), M, Hc, Wc, 64, gains=g)
    ref, ref_mask = EX.feather(frames, M, Hc, Wc, 64, cv)
    assert np.array_equal(out.cpu().numpy(), ref) and np.array_equal(mask.cpu().numpy(), ref_mask)


# ---- a camera-size sweep with known exposures ----------------------------------------------------------------------------------
def _overlap_mad(frames, M, Hc, Wc, gains):
    """Mean absolute difference between the compensated ROI warps of every overlapping pair, over the pixels both cover."""
    take, imgs, masks, tls = EX.fed(frames, M, Hc, Wc)
    imgs = [EX.apply(img, gains[k]) for img, k in zip(imgs, take)]
    tot, cnt = 0.0, 0
    for i, j, (x0, y0, x1, y1) in EX.pairs([(x, y, x + m.shape[1], y + m.shape[0]) for (x, y), m in zip(tls, masks)]):
        if i == j:
            continue
        si = (slice(y0 - tls[i][1], y1 - tls[i][1]), slice(x0 - tls[i][0], x1 - tls[i][0]))
        sj = (slice(y0 - tls[j][1], y1 - tls[j][1]), slice(x0 - tls[j][0], x1 - tls[j][0]))
        both = (masks[i][si] == 255) & (masks[j][sj] == 255)
        tot += np.abs(imgs[i][si][both].astype(np.int64) - imgs[j][sj][both]).sum()
        cnt += 3 * int(both.sum())
    return tot / cnt


def test_known_exposures_are_recovered_on_a_12mp_sweep():
    """Three 3000 x 4000 frames scaled by 0.75, 1.0 and 1.3 (after 0.7, so nothing saturates).  cv2's rule pulls every
    gain towards 1 (beta) and so recovers only part of a step per feed; with four feeds, gain mode recovers the ratios to
    within 1 %.  The compensated overlaps differ less than the raw ones."""
    from unsuperviseddeephomographyral2018_b200 import ops
    e = np.array([0.75, 1.0, 1.3])
    frames, M, (Hc, Wc) = sweep_case(3, 3000, 4000, seed=5, exposures=e)
    g = ops.mosaic_exposure_gains(_cuda(frames), M, Hc, Wc, "gain", 4)
    r = g[:, 0] * e
    print("gains", g[:, 0], "recovered ratio error", np.abs(r / r[1] - 1).max())
    assert np.abs(r / r[1] - 1).max() < 0.01
    before = _overlap_mad(frames, M, Hc, Wc, np.ones((3, 3)))
    after = _overlap_mad(frames, M, Hc, Wc, g)
    print("overlap MAD %.3f -> %.3f" % (before, after))
    assert after < before


# ---- the CLI -------------------------------------------------------------------------------------------------------------------
def test_cli_end_to_end(tmp_path):
    import mosaic_images as cli
    from unsuperviseddeephomographyral2018_b200 import ops
    raw = tmp_path / "raw"
    raw.mkdir()
    frames, _, _ = sweep_case(4, 240, 320, seed=9, exposures=(0.8, 1.0, 1.25, 0.9))
    names = ["DSC_%04d.JPG" % k for k in range(4)]
    for nm, f in zip(names, frames):
        cv2.imwrite(str(raw / nm), f[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, 95])
    out = tmp_path / "mosaic"
    assert cli.main(["--frames", str(raw), "--out_dir", str(out), "--seeded_weights", "True", "--model_dir", str(tmp_path / "none"),
                     "--blend", "multiband", "--compensate", "channels", "--compensate_feeds", "2"]) == 0
    txt = (out / "mosaic.txt").read_text().splitlines()
    head = txt[0].split()
    assert head[0] == "canvas" and head[3] == "ref" and head[5:] == ["blend", "multiband", "5", "compensate", "channels", "2"]
    Hc, Wc = int(head[1]), int(head[2])
    imgs, Ms, gains = [], [], []
    for ln, nm in zip(txt[1:], names):
        parts = ln.split()
        assert parts[0] == nm and parts[1] in ("kept", "dropped") and len(parts) == 14
        if parts[1] == "kept":
            imgs.append(cv2.imread(str(raw / nm))[..., ::-1].copy())
            Ms.append(np.array([float(v) for v in parts[2:11]]).astype(np.float32).astype(np.float64).reshape(3, 3))
            gains.append([float(v) for v in parts[11:]])
    M = np.stack(Ms)
    assert np.array_equal(np.array(gains), EX.gains(imgs, M, Hc, Wc, "channels", 2))
    mos, _ = EX.multiband(imgs, M, Hc, Wc, 5, np.array(gains))
    assert (out / "mosaic.jpg").read_bytes() == ops.encode_jpeg(np.ascontiguousarray(mos[..., ::-1])[None])[0]
