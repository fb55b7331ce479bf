"""CPU checks of oracle/synth_fp32.py, the restatement that tests/test_gpu_input_certify.py holds the input pipeline's
kernels to: the restated fp32 chains against exact rational evaluation in the same order, the keys against a plain
integer splitmix64, and the augmentation table against the project's other restatements of the same definition."""
import decimal
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import draw as D
from oracle import ecc as E
from oracle import oracle as O
from oracle import synth_fp32 as S

f32 = np.float32
M64 = (1 << 64) - 1
SEEDS = [0, 1, 2 ** 63, 2 ** 64 - 1, 0x5DEECE66D]


# ---------------------------------------------------------------------------- exact scalar evaluation
def rf32(q):
    """The fp32 value nearest the rational q (ties to even); normal range only, which is all these chains reach."""
    q = Fraction(q)
    if q == 0:
        return Fraction(0)
    s = -1 if q < 0 else 1
    a = abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    assert -126 <= e < 128, e
    scaled = a / Fraction(2) ** (e - 23)                       # in [2^23, 2^24)
    n, r = divmod(scaled.numerator, scaled.denominator)
    twice = 2 * r
    if twice > scaled.denominator or (twice == scaled.denominator and n % 2 == 1):
        n += 1
    return s * Fraction(n) * Fraction(2) ** (e - 23)


def fr(x):
    return Fraction(float(x))


def py_mix64(x):
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def py_key(seed, b, tag):
    return py_mix64(py_mix64(py_mix64(seed & M64) ^ b) ^ tag)


def py_unit(key):
    return Fraction((py_mix64(key) >> 32) >> 8, 1 << 24) - Fraction(1, 2)


def exact_texture_v(seed, b, c, x, y):
    """texture_u8_kernel's v at one pixel, every operation rounded to fp32 exactly (fma: one rounding)."""
    lat = lambda o, gx, gy: py_unit(py_key(seed, b, c * 6 + o) ^ (gx | (gy << 32)))
    v = lat(0, x, y)
    amp = Fraction(1)
    for o in range(1, 6):
        amp = rf32(amp * fr(f32(1.8660660)))
        fx, fy = rf32(Fraction(x, 1 << o)), rf32(Fraction(y, 1 << o))
        gx, gy = int(fx), int(fy)
        tx, ty = rf32(fx - gx), rf32(fy - gy)
        tx = rf32(rf32(tx * tx) * rf32(3 - rf32(tx + tx)))
        ty = rf32(rf32(ty * ty) * rf32(3 - rf32(ty + ty)))
        a, bb, cc, d = lat(o, gx, gy), lat(o, gx + 1, gy), lat(o, gx, gy + 1), lat(o, gx + 1, gy + 1)
        top = rf32(tx * rf32(bb - a) + a)
        bot = rf32(tx * rf32(d - cc) + cc)
        v = rf32(rf32(ty * rf32(bot - top) + top) * amp + v)
    return v


# ---------------------------------------------------------------------------- keys and draws
@pytest.mark.parametrize("seed", SEEDS)
def test_mix64_and_stream_keys_match_integer_splitmix(seed):
    b = np.array([0, 1, 2, 127, 128, 4095])
    tags = np.arange(28)
    got = S.stream_key(seed, b[:, None], tags[None, :])
    for i, bi in enumerate(b):
        for t in tags:
            assert int(got[i, t]) == py_key(seed, int(bi), int(t)), (seed, bi, t)
    assert int(S.mix64(seed)[0]) == py_mix64(seed & M64)


def test_amplitudes_are_the_constants_ptxas_folded():
    # the FFMA immediates of texture_u8_kernel's octave sum (cuobjdump -sass, sm_90a)
    sass = [1.86606597900390625, 3.4822022914886474609, 6.4980192184448242188, 12.125732421875, 22.627416610717773438]
    assert [float(a) for a in S.AMP] == pytest.approx(sass, rel=0, abs=1e-15)


@pytest.mark.parametrize("seed", SEEDS)
def test_texture_restatement_equals_exact_evaluation(seed):
    Hh, W = 67, 93                                   # ragged: partial octave cells at both edges
    rng = np.random.default_rng(seed & 0xFFFF)
    for b in (0, 1, 127):
        img = S.texture(seed, b, Hh, W)
        pts = [(0, 0), (W - 1, Hh - 1), (31, 31), (32, 32), (33, 15)] + [(int(p[0]), int(p[1])) for p in rng.integers(0, (W, Hh), size=(12, 2))]
        for c in range(3):
            vs = S.texture_v(seed, b, c, Hh, W)
            for x, y in pts:
                v = exact_texture_v(seed, b, c, x, y)
                assert fr(vs[y, x]) == v, (seed, b, c, x, y, float(vs[y, x]), float(v))
                u = min(max(rf32(v * fr(f32(9.8)) + Fraction(255, 2)), 0), 255)
                assert int(img[y, x, c]) == int(u), (seed, b, c, x, y)


@pytest.mark.parametrize("seed", SEEDS)
def test_corners_are_the_keyed_draws_in_range(seed):
    B, Hh, W, P, rho = 300, 240, 320, 128, 45
    pts1, gt = S.corners(seed, B, Hh, W, P, rho)
    for b in (0, 1, 150, 299):
        draw = lambda i: (py_mix64(py_key(seed, b, S.TAG_CORNERS + i)) >> 32)
        x0, y0 = rho + draw(0) % (W - 2 * rho - P + 1), rho + draw(1) % (Hh - 2 * rho - P + 1)
        assert list(pts1[b]) == [x0, y0, x0 + P, y0, x0 + P, y0 + P, x0, y0 + P]
        assert list(gt[b]) == [draw(2 + i) % (2 * rho + 1) - rho for i in range(8)]
    assert pts1[:, 0].min() >= rho and pts1[:, 0].max() <= W - rho - P
    assert pts1[:, 1].min() >= rho and pts1[:, 1].max() <= Hh - rho - P
    assert np.abs(gt).max() <= rho


def test_adjacent_seeds_and_samples_draw_unrelated_values():
    """The defect the keys fix: seed s and s ^ 1 (the dataloader's consecutive steps) must not shift each other's draws."""
    B = 8
    for s in (0, 2, 1000002):
        _, g0 = S.corners(s, B, 240, 320, 128, 45)
        _, g1 = S.corners(s + 1, B, 240, 320, 128, 45)
        for k in range(1, 8):
            assert not np.array_equal(g1[:, :8 - k], g0[:, k:])


# ---------------------------------------------------------------------------- the augmentation table
def exact_pow_f32(x, g):
    with decimal.localcontext() as ctx:
        ctx.prec = 60
        p = decimal.Decimal(x) ** decimal.Decimal(float(f32(g))) if x else decimal.Decimal(0)
        return rf32(Fraction(p))


AUG_ROWS = [
    [1, 1.0, 1.0, 1.0, 1.0, 1.0, 1, 1.0, 1.0, 1.0, 1.0, 1.0],       # gamma 1 exactly, unit gains: the identity
    [1, 1.2, 2.0, 1.2, 1.2, 1.2, 1, 0.8, 0.5, 0.8, 0.8, 0.8],       # saturates at 255 / darkens
    [1, 0.9137, 1.37, 1.05, 0.83, 1.19, 1, 1.1712, 0.61, 0.97, 1.13, 0.88],
    [1, 1.0, 0.0, 1.0, -0.5, 1.0, 1, 1.07, 1.0, 0.0, 1.0, -1.0],    # to 0 (zero brightness, negative and zero gains)
]


@pytest.mark.parametrize("row", range(len(AUG_ROWS)))
def test_table_equals_exact_evaluation(row):
    aug = np.asarray(AUG_ROWS[row][:11], f32)
    L = S.tables(aug)
    for im in range(2):
        a = aug[1 + 5 * im:6 + 5 * im]
        for x in range(256):
            p = exact_pow_f32(x, a[0])
            for c in range(3):
                v = rf32(rf32(p * fr(a[1])) * fr(a[2 + c]))
                v = min(max(v, 0), 255)
                n = rf32(rf32(v - fr(S.MEAN[c])) / fr(S.STD[c]))
                assert fr(L[im, c, x]) == n, (row, im, c, x)


@pytest.mark.parametrize("row", range(len(AUG_ROWS)))
def test_table_equals_the_ecc_and_report_restatements(row):
    """oracle/ecc.py and oracle/draw.py define the augmentation the same way: the tables are identical bit for bit."""
    aug = np.asarray(AUG_ROWS[row][:11], f32)
    L = S.tables(aug)
    img = np.stack([np.arange(256, dtype=np.uint8)] * 3, 1)[None]     # [1, 256, 3]: every value in every channel
    for im in range(2):
        n = E.augment_normalise(img, aug[1 + 5 * im:6 + 5 * im])[0]
        assert np.array_equal(n, L[im].T), (row, im)
        assert np.array_equal(D.host_denorm(img, aug, im)[0], E.denorm_u8(L[im].T[None])[0]), (row, im)
    assert np.array_equal(S.tables(None)[0].T, E.augment_normalise(img, None)[0])


@pytest.mark.parametrize("row", range(len(AUG_ROWS)))
def test_table_within_the_pow_definition_of_oracle_prep_inputs(row):
    """oracle.prep_inputs raises to gamma with torch's fp32 pow, which is not correctly rounded: the two tables differ by
    at most what a few ulps of the power become through the gains and the normalisation."""
    aug = np.asarray(AUG_ROWS[row][:11], f32)
    L = S.tables(aug)
    img = np.stack([np.arange(256, dtype=np.uint8)] * 3, 1).reshape(16, 16, 3)
    ref = O.prep_inputs(torch.tensor(img[None]), torch.tensor(img[None]), torch.zeros(1, 8), torch.tensor(aug[None]), 16)
    for im, key in ((0, "I_aug"), (1, "I_prime_aug")):
        r = ref[key][0].numpy().reshape(256, 3).T
        a = aug[1 + 5 * im:6 + 5 * im]
        p = np.power(np.arange(256, dtype=np.float64), np.float64(a[0]))
        g = np.abs(a[1:2] * a[2:5])[:, None]
        bound = (4 * 2.0 ** -24 * p * g + 4 * 2.0 ** -24 * (np.minimum(p * g, 255) + S.MEAN[:, None])) / S.STD[:, None]
        assert np.all(np.abs(r.astype(np.float64) - L[im]) <= bound), (row, im)


def test_pow_f32_guard_fires():
    # no uint8 power is known to sit within 64 fp64 ulps of an fp32 boundary; a huge margin makes the guard fire
    with pytest.raises(AssertionError):
        S.pow_f32(np.arange(256), f32(1.1), margin_ulps=2 ** 40)


# ---------------------------------------------------------------------------- gathers and the float4 phase
def test_normalise_u8_phase_equals_per_element_channel():
    rng = np.random.default_rng(3)
    for n in (12, 16, 20, 24, 3 * 4 * 7 * 11):
        u = rng.integers(0, 256, size=n, dtype=np.uint8)
        ch = np.arange(n) % 3
        ref = ((u.astype(f32) - S.MEAN[ch]).astype(f32) / S.STD[ch]).astype(f32)
        assert np.array_equal(S.normalise_u8(u), ref), n


def test_prep_ex_restatement_against_oracle_prep_inputs():
    rng = np.random.default_rng(7)
    B, Hh, W, P = 4, 37, 45, 16
    I = rng.integers(0, 256, size=(B, Hh, W, 3), dtype=np.uint8)
    Ip = rng.integers(0, 256, size=(B, Hh, W, 3), dtype=np.uint8)
    x0 = np.array([0, W - P, 0, 13]); y0 = np.array([0, Hh - P, Hh - P, 5])
    pts1 = np.stack([x0, y0, x0 + P, y0, x0 + P, y0 + P, x0, y0 + P], 1).astype(f32)
    aug = np.asarray([AUG_ROWS[2][:11], [0] * 11, AUG_ROWS[1][:11], AUG_ROWS[3][:11]], f32)
    got = S.prep_ex(I, Ip, pts1, aug, P)
    ref = O.prep_inputs(torch.tensor(I), torch.tensor(Ip), torch.tensor(pts1), torch.tensor(aug), P)
    assert np.array_equal(got["origin"], ref["patch_indices"][:, 0].numpy())
    for k in ("I1", "I2"):                                    # no pow: the same sums, to the rounding of torch's mean
        assert np.abs(got[k] - ref[k].numpy()).max() <= 2 * 2.0 ** -23 * 3, k
    for k in ("I1_aug", "I2_aug"):
        assert np.abs(got[k] - ref[k].numpy()).max() <= 1e-5, k
    assert np.abs(got["I_aug3"] - ref["I_aug"].numpy()).max() <= 1e-5
    I1, I2, org = S.patches_u8(I, Ip, pts1, P)
    assert np.array_equal(I1, got["I1"][..., 0]) and np.array_equal(I2, got["I2"][..., 0])
    assert np.array_equal(org, got["origin"])
    # sample 1 is not augmented: its augmented outputs are the plain ones
    assert np.array_equal(got["I1_aug"][1], got["I1"][1]) and np.array_equal(got["I2_aug"][1], got["I2"][1])
