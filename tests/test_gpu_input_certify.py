"""The train step's device input pipeline, bit for bit against oracle/synth_fp32.py (checked on the CPU by
tests/test_input_certify_logic.py): udh_synth_scene_u8 (texture_u8_kernel, corners_kernel), udh_prep_inputs_u8_ex
(prep_u8_ex_kernel) and udh_prep_inputs_u8 (normalise_u8_kernel, patches_u8_kernel); the statistics of the draws over the
dataloader's own seed sequence; the augmentation across the prep and ECC paths; and synthetic.make_batch_fast end to end.
A failure names the kernel, the output and the first differing element."""
import ctypes

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import ecc as E
from oracle import synth_fp32 as S

pytestmark = pytest.mark.gpu
f32 = np.float32
P, RHO = 128, 45


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from unsuperviseddeephomographyral2018_b200 import _lib
    return _lib


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _same(kernel, name, got, ref):
    """Bit-identical (NaN never matches): on failure, the kernel, the output and the first differing index."""
    got = np.asarray(got); ref = np.asarray(ref)
    assert got.shape == ref.shape, (kernel, name, got.shape, ref.shape)
    bad = got.view(np.uint8 if got.dtype == np.uint8 else np.int32) != ref.view(np.uint8 if ref.dtype == np.uint8 else np.int32)
    if bad.any():
        i = tuple(int(v) for v in np.argwhere(bad)[0])
        pytest.fail("%s: %s differs at %d of %d elements; first at %s: got %r, restated %r"
                    % (kernel, name, int(bad.sum()), bad.size, i, got[i], ref[i]))


def _scene(L, B, Hh, W, seed):
    I = torch.empty(B, Hh, W, 3, device="cuda", dtype=torch.uint8)
    pts1 = torch.empty(B, 8, device="cuda"); gt = torch.empty(B, 8, device="cuda")
    L.check(L.lib.udh_synth_scene_u8(_p(I), _p(pts1), _p(gt), B, Hh, W, P, RHO, seed, None), "udh_synth_scene_u8")
    torch.cuda.synchronize()
    return I, pts1, gt


# ---------------------------------------------------------------------------- scene
@pytest.mark.parametrize("seed", [0, 1, 2 ** 63, 2 ** 64 - 1])
@pytest.mark.parametrize("size", [(240, 320), (241, 333)], ids=["240x320", "241x333"])
@pytest.mark.parametrize("B", [1, 3, 128])
def test_scene_bit_identical(L, B, size, seed):
    Hh, W = size
    I, pts1, gt = _scene(L, B, Hh, W, seed)
    samples = range(B) if B <= 3 else (0, 1, 63, 64, 126, 127)
    ref_img, ref_pts, ref_gt = S.scene(seed, B, Hh, W, P, RHO, samples)
    _same("corners_kernel", "pts1", pts1.cpu().numpy(), ref_pts)
    _same("corners_kernel", "gt", gt.cpu().numpy(), ref_gt)
    got = I.cpu().numpy()
    for b in samples:
        _same("texture_u8_kernel", "I[b=%d]" % b, got[b], ref_img[b])


def test_scene_draws_cover_their_ranges(L):
    """Over 16 384 samples every x0 and y0 of the range is drawn, and x0, y0 and gt's 91 values pass a chi-squared test."""
    x0s, y0s, gts = [], [], []
    for seed in range(8):
        _, pts1, gt = _scene(L, 2048, 240, 320, 1000 + seed)
        x0s.append(pts1[:, 0].cpu().numpy()); y0s.append(pts1[:, 1].cpu().numpy()); gts.append(gt.cpu().numpy().ravel())
    for name, v, lo, hi in (("x0", np.concatenate(x0s), RHO, 320 - RHO - P), ("y0", np.concatenate(y0s), RHO, 240 - RHO - P),
                            ("gt", np.concatenate(gts), -RHO, RHO)):
        assert np.all(v == np.round(v)) and v.min() >= lo and v.max() <= hi, name
        counts = np.bincount((v - lo).astype(np.int64), minlength=hi - lo + 1)
        assert counts.min() > 0, (name, "values never drawn", np.nonzero(counts == 0)[0] + lo)
        p = stats.chisquare(counts).pvalue
        print("\n  %s: %d draws over %d values, chi-squared p = %.3f" % (name, v.size, counts.size, p))
        assert p > 1e-6, (name, p)


def test_consecutive_steps_and_samples_are_independent(L):
    """The dataloader's synthetic batches over 400 steps (seed * 1000003 + step, consecutive seeds one apart): no sample's
    gt is a shift of another sample's (overlaps of 5 to 8 draws), and the pixel correlation between the same sample of
    steps s and s + 1, and between samples b and b + 1 of one batch, sits at the level of independent scenes, measured by
    the same correlation with one of the two images turned by 180 degrees."""
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl
    B, steps = 16, 400
    dparams = dl.dataloader_params(data_path="", filenames_file=None, pts1_file=None, gt_file=None, mode='train', batch_size=B,
                                   img_h=240, img_w=320, patch_size=P, augment_list=['normalize'], do_augment=0.0)
    loader = dl.Dataloader(dparams, shuffle=True, synthetic_pairs=B * steps, seed=0, device="cuda")
    gts = np.empty((steps, B, 8), np.int64)
    adj, adj_ctl, inb, inb_ctl = [], [], [], []
    prev = None
    for s in range(steps):
        b = loader.next_batch()
        gts[s] = b["gt"].cpu().numpy().astype(np.int64)
        z = b["I_u8"].float().reshape(B, -1)
        z = (z - z.mean(1, keepdim=True)) / z.std(1, correction=0, keepdim=True)
        z = z.reshape(B, 240, 320, 3)
        rot = torch.flip(z, dims=(1, 2))
        inb.append((z[:-1] * z[1:]).mean(dim=(1, 2, 3))); inb_ctl.append((z[:-1] * rot[1:]).mean(dim=(1, 2, 3)))
        if prev is not None:
            adj.append((prev[0] * z).mean(dim=(1, 2, 3))); adj_ctl.append((prev[0] * rot).mean(dim=(1, 2, 3)))
        prev = (z,)
    # shifted draws: a window of n >= 5 consecutive gt values of one sample equal to the first n of another
    seen = {}
    flat = gts.reshape(-1, 8)
    for i, g in enumerate(flat):
        for n in (8, 7, 6, 5):
            seen.setdefault((n, tuple(g[:n])), []).append(i)
    for i, g in enumerate(flat):
        for k in range(0, 4):
            for j in seen.get((8 - k, tuple(g[k:])), []):
                assert k == 0 and j == i, ("corners_kernel: gt of step %d sample %d from draw %d on equals the first %d draws of step %d "
                                           "sample %d" % (i // B, i % B, k, 8 - k, j // B, j % B))
    rms = lambda v: float(torch.sqrt((torch.cat(v) ** 2).mean()))
    for name, c, ctl in (("steps s, s + 1", adj, adj_ctl), ("samples b, b + 1", inb, inb_ctl)):
        cc = torch.cat(c)
        m, r, r0 = float(cc.mean()), rms(c), rms(ctl)
        print("\n  texture_u8_kernel, %s: %d pairs, mean correlation %+.4f, rms %.4f (turned: rms %.4f)" % (name, cc.numel(), m, r, r0))
        assert abs(m) <= 5 * r0 / np.sqrt(cc.numel()) and r <= 1.25 * r0, ("texture_u8_kernel: scenes of %s are correlated" % name, m, r, r0)


# ---------------------------------------------------------------------------- fused prep
def _images(rng, B, Hh, W):
    I = rng.integers(0, 256, size=(B, Hh, W, 3), dtype=np.uint8)
    Ip = rng.integers(0, 256, size=(B, Hh, W, 3), dtype=np.uint8)
    return I, Ip


def _origins(rng, B, Hh, W, p=P):
    """Window origins of p x p patches: the four extreme corners first, then random."""
    x0 = rng.integers(0, W - p + 1, size=B); y0 = rng.integers(0, Hh - p + 1, size=B)
    for i, (x, y) in enumerate([(0, 0), (W - p, 0), (0, Hh - p), (W - p, Hh - p)][:B]):
        x0[i], y0[i] = x, y
    return np.stack([x0, y0, x0 + p, y0, x0 + p, y0 + p, x0, y0 + p], 1).astype(f32)


def _five(rng, n):
    return np.concatenate([rng.uniform(0.8, 1.2, (n, 1)), rng.uniform(0.5, 2.0, (n, 1)), rng.uniform(0.8, 1.2, (n, 3))], 1)


EDGE_ROWS = np.array([
    [1, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0],          # gamma 1, unit gains: equal to the plain path
    [1, 1.2, 2.0, 1.2, 1.2, 1.2, 1.2, 2.0, 1.2, 1.2, 1.2],          # saturates at 255
    [1, 0.8, 0.5, 0.8, 0.8, 0.8, 1.0, 0.0, 1.0, 1.0, 1.0],          # dark; I' to 0 (zero brightness)
    [1, 1.0, 1.0, 1.0, -0.5, 1.0, 1.13, 1.0, 0.0, 1.0, -1.0],       # negative and zero gains: clipped to 0
], f32)


def _aug(kind, B, rng):
    if kind == "null":
        return None
    a = np.zeros((B, 11), f32)
    a[:, 0] = 1
    if kind in ("mixed", "joint", "disjoint"):
        five = _five(rng, B)
        a[:, 1:6] = five
        a[:, 6:11] = five if kind != "disjoint" else _five(rng, B)
        if kind == "mixed":
            a[1::2, 0] = 0                                              # every other sample not augmented
            a[np.arange(B) % 3 == 0, 6:11] = _five(rng, (np.arange(B) % 3 == 0).sum())   # some rows disjoint
    elif kind == "edge":
        a[:] = EDGE_ROWS[np.arange(B) % len(EDGE_ROWS)]
    return a


def _prep_ex(L, I, Ip, pts1, aug, outs=("gray", "rgb", "plain"), p=P):
    B, Hh, W, _ = I.shape
    d = lambda *s: torch.full(s, float("nan"), device="cuda")
    t = lambda a: torch.tensor(a).cuda() if a is not None else None
    I_d, Ip_d, pts_d, aug_d = t(I), t(Ip), t(pts1), t(aug)
    o = dict(I_gray=d(B, Hh, W, 1) if "gray" in outs else None, I_aug3=d(B, Hh, W, 3) if "rgb" in outs else None,
             I1=d(B, p, p, 1) if "plain" in outs else None, I2=d(B, p, p, 1) if "plain" in outs else None,
             I1_aug=d(B, p, p, 1), I2_aug=d(B, p, p, 1), origin=torch.full((B,), -7, device="cuda", dtype=torch.int32))
    L.check(L.lib.udh_prep_inputs_u8_ex(_p(I_d), _p(Ip_d), _p(pts_d), _p(aug_d), _p(o["I_gray"]), _p(o["I_aug3"]), _p(o["I1"]),
                                        _p(o["I2"]), _p(o["I1_aug"]), _p(o["I2_aug"]), _p(o["origin"]), B, Hh, W, p, None),
            "udh_prep_inputs_u8_ex")
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items() if v is not None}


def _check_prep_ex(got, ref):
    for k, v in got.items():
        _same("prep_u8_ex_kernel", k, v, ref[k])


@pytest.mark.parametrize("kind", ["null", "mixed", "joint", "disjoint", "edge"])
@pytest.mark.parametrize("B", [1, 5, 128, 129])
def test_prep_ex_bit_identical(L, B, kind):
    rng = np.random.default_rng(B * 10 + len(kind))
    I, Ip = _images(rng, B, 240, 320)
    pts1 = _origins(rng, B, 240, 320)
    aug = _aug(kind, B, rng)
    _check_prep_ex(_prep_ex(L, I, Ip, pts1, aug), S.prep_ex(I, Ip, pts1, aug, P))


@pytest.mark.parametrize("size", [(241, 333), (131, 129), (128, 128), (600, 500)], ids=lambda s: "%dx%d" % s)
def test_prep_ex_ragged_sizes(L, size):
    """Pixel counts that are not a multiple of the grid stride (256 threads x min(ceil(h w / 1024), 256) CTAs), one that
    needs the full 256-CTA stride several times (600 x 500), and the patch filling the image (128 x 128)."""
    Hh, W = size
    B = 5
    rng = np.random.default_rng(Hh * W)
    I, Ip = _images(rng, B, Hh, W)
    pts1 = _origins(rng, B, Hh, W)
    aug = _aug("mixed", B, rng)
    _check_prep_ex(_prep_ex(L, I, Ip, pts1, aug), S.prep_ex(I, Ip, pts1, aug, P))


@pytest.mark.parametrize("outs", [("gray",), ("rgb",), ("gray", "rgb"), ("gray", "plain"), ("rgb", "plain"), ("gray", "rgb", "plain")],
                         ids=lambda o: "+".join(o))
def test_prep_ex_optional_outputs(L, outs):
    B = 5
    rng = np.random.default_rng(len(outs) * 7 + len(outs[0]))
    I, Ip = _images(rng, B, 241, 333)
    pts1 = _origins(rng, B, 241, 333)
    aug = _aug("mixed", B, rng)
    _check_prep_ex(_prep_ex(L, I, Ip, pts1, aug, outs), S.prep_ex(I, Ip, pts1, aug, P))


@pytest.mark.parametrize("swap", [False, True], ids=["I", "I_prime"])
def test_prep_ex_every_table_entry(L, swap):
    """Every entry of both images' tables is read: I_aug3 holds I's table at every uint8 value of every channel; with the
    images and the two halves of each row swapped it holds I''s."""
    B = 8
    rng = np.random.default_rng(11)
    I, Ip = _images(rng, B, 130, 136)
    aug = np.concatenate([_aug("disjoint", 4, rng), EDGE_ROWS])
    if swap:
        I, Ip = Ip, I
        aug = np.concatenate([aug[:, :1], aug[:, 6:11], aug[:, 1:6]], 1)
    for b in range(B):
        for c in range(3):
            assert np.unique(I[b, ..., c]).size == 256
    pts1 = _origins(rng, B, 130, 136)
    _check_prep_ex(_prep_ex(L, I, Ip, pts1, aug), S.prep_ex(I, Ip, pts1, aug, P))


# ---------------------------------------------------------------------------- plain prep
def _plain_sizes():
    """(B, h, w) with B h w 3 = 0, 4, 8 and 12 mod 16: the last float4 starts at each channel phase."""
    out = {}
    for B in (1, 3):
        for h in range(128, 150):
            for w in range(128, 150):
                r = B * h * w * 3 % 16
                if r % 4 == 0 and r not in out:
                    out[r] = (B, h, w)
    return [out[r] for r in (0, 4, 8, 12)]


@pytest.mark.parametrize("shape", _plain_sizes(), ids=lambda s: "B%d_%dx%d_mod16_%d" % (s + (s[0] * s[1] * s[2] * 3 % 16,)))
def test_prep_plain_bit_identical(L, shape):
    B, Hh, W = shape
    rng = np.random.default_rng(Hh + W)
    I, Ip = _images(rng, B, Hh, W)
    pts1 = _origins(rng, B, Hh, W)
    t = lambda a: torch.tensor(a).cuda()
    I_d, Ip_d, pts_d = t(I), t(Ip), t(pts1)
    I_aug = torch.full((B, Hh, W, 3), float("nan"), device="cuda")
    I1 = torch.full((B, P, P), float("nan"), device="cuda"); I2 = torch.full_like(I1, float("nan"))
    org = torch.full((B,), -7, device="cuda", dtype=torch.int32)
    L.check(L.lib.udh_prep_inputs_u8(_p(I_d), _p(Ip_d), _p(pts_d), _p(I_aug), _p(I1), _p(I2), _p(org), B, Hh, W, P, None), "udh_prep_inputs_u8")
    torch.cuda.synchronize()
    _same("normalise_u8_kernel", "I_aug", I_aug.cpu().numpy().reshape(-1), S.normalise_u8(I))
    r1, r2, ro = S.patches_u8(I, Ip, pts1, P)
    _same("patches_u8_kernel", "I1", I1.cpu().numpy(), r1)
    _same("patches_u8_kernel", "I2", I2.cpu().numpy(), r2)
    _same("patches_u8_kernel", "origin", org.cpu().numpy(), ro)


# ---------------------------------------------------------------------------- across paths
def test_augmentation_agrees_with_the_ecc_tables(L):
    """One augmentation row gives the same augmented values in udh_prep_inputs_u8_ex as in udh_ecc_prep_u8: the prep's
    normalised values (I_aug3, and with the roles swapped I''s), denormalised and made gray on the host, equal the ECC
    path's gray planes on images holding every value of every channel."""
    from unsuperviseddeephomographyral2018_b200 import ops
    B, Hh, W = 24, 64, 64
    rng = np.random.default_rng(23)
    I, Ip = _images(rng, B, Hh, W)
    aug = np.concatenate([_aug("disjoint", B - len(EDGE_ROWS), rng), EDGE_ROWS])
    g1, g2 = ops.ecc_prep_u8(torch.tensor(I).cuda(), torch.tensor(Ip).cuda(), torch.tensor(aug).cuda())
    pts1 = _origins(rng, B, Hh, W, 16)
    a = _prep_ex(L, I, Ip, pts1, aug, ("rgb",), 16)["I_aug3"]
    swapped = np.concatenate([aug[:, :1], aug[:, 6:11], aug[:, 1:6]], 1)
    b = _prep_ex(L, Ip, I, pts1, swapped, ("rgb",), 16)["I_aug3"]
    _same("prep_u8_ex_kernel", "I_aug3", a, S.prep_ex(I, Ip, pts1, aug, 16)["I_aug3"])
    for name, n, g in (("gray_I", a, g1), ("gray_I_prime", b, g2)):
        host = np.stack([E.rgb2gray_u8(E.denorm_u8(n[i])) for i in range(B)])
        _same("prep_u8_ex_kernel vs ecc_prep_kernel", name, host, g.cpu().numpy().reshape(B, Hh, W))


# ---------------------------------------------------------------------------- end to end
def test_make_batch_fast_equals_the_chain(L):
    """make_batch_fast at B = 128 equals the chain of restatements: the scene, then the device DLT and udh_warp_image_u8
    (certified in test_gpu_photometric.py) on the restated scene, then the restated fused prep."""
    from unsuperviseddeephomographyral2018_b200 import ops, synthetic
    B, seed = 128, 20261018
    out = synthetic.make_batch_fast(B, seed=seed, do_augment=0.5, want_rgb=True)
    torch.cuda.synchronize()
    imgs, pts1, gt = S.scene(seed, B, 240, 320, P, RHO)
    I_ref = np.stack([imgs[b] for b in range(B)])
    _same("texture_u8_kernel", "I_u8", out["I_u8"].cpu().numpy(), I_ref)
    _same("corners_kernel", "pts1", out["pts1"].cpu().numpy(), pts1)
    _same("corners_kernel", "gt", out["gt"].cpu().numpy(), gt)
    I_d = torch.tensor(I_ref).cuda()
    H = ops.dlt_forward(torch.tensor(pts1).cuda(), torch.tensor(gt).cuda()).reshape(B, 9).contiguous()
    Ip_d = torch.empty_like(I_d)
    L.check(L.lib.udh_warp_image_u8(_p(I_d), _p(H), _p(Ip_d), B, 240, 320, None), "udh_warp_image_u8")
    Ip_ref = Ip_d.cpu().numpy()
    _same("udh_warp_image_u8", "I_prime_u8", out["I_prime_u8"].cpu().numpy(), Ip_ref)
    gen = torch.Generator(device="cuda"); gen.manual_seed(seed * 7919 + 13)
    aug = synthetic.draw_augmentation(B, 0.5, "train", gen, torch.device("cuda")).cpu().numpy()
    assert np.array_equal(out["aug"].cpu().numpy(), aug) and 0 < aug[:, 0].sum() < B
    ref = S.prep_ex(I_ref, Ip_ref, pts1, aug, P)
    for k, r in (("I1", "I1"), ("I2", "I2"), ("I1_aug", "I1_aug"), ("I2_aug", "I2_aug"), ("I_aug", "I_gray"), ("I_aug_rgb", "I_aug3"),
                 ("patch_indices", "origin")):
        _same("make_batch_fast", k, out[k].cpu().numpy(), ref[r])
