"""CPU tests of oracle/x3_limbs.py, the restatement of the two-limb format that tests/test_gpu_x3_certify.py holds the kernels
to: split and join against exact rational evaluation (including the midpoint case where a re-split changes the limbs but
not the value), the exactness precondition of every operand generator at the largest K of each instance, and the
per-element bound against an exact evaluation of three-pass dot products accumulated the way a wgmma chain may round."""
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import x3_limbs as X

f32 = np.float32


def rn(q, p):
    """Fraction -> nearest value with p significant bits, ties to even (normal range)."""
    if q == 0:
        return Fraction(0)
    a = abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    quantum = Fraction(2) ** (e - p + 1)
    r = round(a / quantum) * quantum                        # Fraction.__round__: half to even
    return r if q > 0 else -r


def trunc(q, p=24):
    """Fraction -> p significant bits, toward zero."""
    if q == 0:
        return Fraction(0)
    a = abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    quantum = Fraction(2) ** (e - p + 1)
    r = (a // quantum) * quantum
    return r if q > 0 else -r


def exact_split(x):
    hi = rn(Fraction(float(x)), 8)
    return hi, rn(Fraction(float(x)) - hi, 8)


def _values(seed, n=4000):
    rng = np.random.default_rng(seed)
    wide = np.exp2(rng.uniform(-24, 0, n)) * np.where(rng.random(n) < 0.5, -1, 1)
    return np.concatenate([rng.standard_normal(n), wide, rng.standard_normal(n) * 1e3, [0.0, -0.0, 1.0, 255.5]]).astype(f32)


def test_split_and_join_equal_exact_rounding():
    v = _values(0)
    hi, lo = X.split(torch.tensor(v))
    j = X.join(hi, lo)
    for i, x in enumerate(v):
        eh, el = exact_split(x)
        assert Fraction(float(hi[i])) == eh and Fraction(float(lo[i])) == el, (x, float(hi[i]), float(lo[i]))
        assert Fraction(float(j[i])) == rn(eh + el, 24)
        assert abs(Fraction(float(j[i])) - Fraction(float(x))) <= Fraction(2) ** -16 * abs(Fraction(float(x)))
    assert torch.equal(X.stored(torch.tensor(v), "bf16"), torch.tensor(v).to(torch.bfloat16).float())
    # stored() is monotone, so a maximum of the fp32 accumulators is a maximum of the stored values (the fused pool1 rule)
    s = torch.sort(torch.tensor(v)).values
    st = X.stored(s)
    assert (st[1:] >= st[:-1]).all()


def test_resplit_midpoint_keeps_the_value_not_the_limbs():
    """x - hi rounds UP to exactly half an ulp of an odd hi: the joined value is a bf16 midpoint, and splitting it again
    rounds the tie to the even neighbour of hi, with the negative half ulp as lo."""
    x = torch.tensor([1 + 2.0 ** -7 + 2.0 ** -8 - 2.0 ** -20], dtype=torch.float32)
    hi, lo = X.split(x)
    assert hi.item() == 1 + 2.0 ** -7 and lo.item() == 2.0 ** -8           # hi odd (last of 8 bits set), lo = half its ulp
    v = X.join(hi, lo)
    h2, l2 = X.split(v)
    assert h2.item() == 1 + 2.0 ** -6 and l2.item() == -2.0 ** -8           # other limbs ...
    assert torch.equal(X.join(h2, l2), v) and torch.equal(X.stored(v), v)  # ... same value: stored() is idempotent
    # the case is not rare on continuous data
    v = torch.tensor(_values(1))
    s = X.stored(v)
    changed = ~(X.split(s)[0] == X.split(v)[0])
    assert torch.equal(X.stored(s), s) and int(changed.sum()) > 0


def test_three_pass_excludes_lo_lo():
    gen = torch.Generator().manual_seed(3)
    x = X.limb_operand(gen, (50,), True, device="cpu")
    w = X.limb_operand(gen, (50,), True, device="cpu")
    got = X.three_pass(lambda a, b: (a * b).sum(), x, w).item()
    want = sum(Fraction(float(h)) * Fraction(float(k)) + Fraction(float(h)) * Fraction(float(l2)) + Fraction(float(l)) * Fraction(float(k))
               for (h, l), (k, l2) in zip(zip(*X.split(x)), zip(*X.split(w))))
    assert Fraction(got) == want


# instances at their largest K: (what, x shape, w shape or None for a weight gradient, x vmax, w vmax, grid, lo on x, on w)
def _conv_abs(x, w):
    return F.conv2d(x.double().abs().permute(0, 3, 1, 2), w.double().abs().permute(3, 2, 0, 1), padding=1)


@pytest.mark.parametrize("cin,cout", [(64, 64), (64, 128), (128, 128)])
def test_conv_generators_are_exact_at_the_largest_k(cin, cout):
    """The forward / dgrad operands of test_gpu_x3_certify.py at K = 9 cin (and 9 cout): integers in -2..2 with an integer
    bias in -3..3, and limb operands (x hi in +-1..2, w hi in +-1, lo on either or both) with a bias in -2..2."""
    gen = torch.Generator().manual_seed(cin + cout)
    for kin in {cin, cout}:
        x = X.int_operand(gen, (1, 16, 16, kin), device="cpu"); w = X.int_operand(gen, (3, 3, kin, 64), device="cpu")
        assert X.require_exact(_conv_abs(x, w) + 3, 1.0, "integer") <= 9 * kin * 4 + 3
        for lx, lw in ((True, False), (False, True), (True, True)):
            x = X.limb_operand(gen, (1, 16, 16, kin), lx, vmax=2, device="cpu"); w = X.limb_operand(gen, (3, 3, kin, 64), lw, vmax=1, device="cpu")
            worst = X.require_exact(_conv_abs(x, w) + 2, X.GRID_LO, "limb")
            # the worst case of any draw (every |x| = 2 + 2^-10, |w| = 1 + 2^-10) is below 2^22 grid units too
            assert (9 * kin * (2 + X.GRID_LO) * (1 + X.GRID_LO) + 2) / X.GRID_LO < X.EXACT_UNITS and worst > 0


@pytest.mark.parametrize("B,H,C", [(128, 128, 64), (70, 128, 64), (128, 16, 128), (70, 32, 128)])
def test_wgrad_generators_are_exact_at_the_largest_k(B, H, C):
    """Integer weight-gradient operands in {-1, 0, 1}: sum |x g| <= B H W = 2^21 at B = 128.  Limb operands: x hi in +-1
    dense, g sparse at density 1024 / (1.5 B H W), so sum |g| (and sum |x g| <= (1 + 2^-10) sum |g|) stays below 2^22 grid
    units (checked on 8 channels of a real draw)."""
    assert B * H * H <= 2 ** 21 < X.EXACT_UNITS
    gen = torch.Generator().manual_seed(B + H)
    g = X.limb_operand(gen, (B, H, H, 8), True, vmax=1, density=min(1.0, 1024.0 / (1.5 * B * H * H)), device="cpu")
    s = g.abs().double().sum(dim=(0, 1, 2))
    X.require_exact(s * (1 + X.GRID_LO), X.GRID_LO, "limb wgrad")
    assert (s > 0).all()


def _x3_dot_chain(x, w, bias, rng):
    """One output of a two-limb kernel, exactly: the hh, hl, lh products of every k16 step of each pass added to the fp32
    accumulator in a random order with truncation (a wgmma's internal order and alignment are unspecified), the bias added,
    the result split and joined (the stored output).  x, w: fp32 arrays of one dot product (K a multiple of 16)."""
    sx = [exact_split(v) for v in x]
    sw = [exact_split(v) for v in w]
    acc = Fraction(0)
    for hx, hw in ((0, 0), (0, 1), (1, 0)):
        for k0 in range(0, len(x), 16):
            terms = [sx[i][hx] * sw[i][hw] for i in range(k0, k0 + 16)]
            for t in rng.permutation(len(terms)):
                acc = trunc(acc + terms[t])
    v = trunc(acc + Fraction(float(bias)))
    hi = rn(v, 8)
    return rn(hi + rn(v - hi, 8), 24)


@pytest.mark.parametrize("kind", ["randn", "wide"])
@pytest.mark.parametrize("K", [32, 576, 1152, 16384])
def test_bound_holds_against_exact_evaluation(K, kind):
    """conv1_1 (K = 18, padded to 32), the 64- and 128-channel convolutions, and a weight-gradient chain of 16384 positions:
    the stored result of a truncating chain lies within X.bound of the exact value of sum x w + b."""
    rng = np.random.default_rng(K + len(kind))
    trials = 3 if K > 2000 else 12
    worst = 0.0
    for _ in range(trials):
        if kind == "randn":
            x, w = rng.standard_normal(K).astype(f32), (rng.standard_normal(K) * 0.05).astype(f32)
        else:
            x = (np.exp2(rng.uniform(-24, 0, K)) * np.where(rng.random(K) < 0.5, -1, 1)).astype(f32)
            w = (np.exp2(rng.uniform(-24, 0, K)) * np.where(rng.random(K) < 0.5, -1, 1)).astype(f32)
        b = f32(rng.standard_normal() * 0.1)
        got = _x3_dot_chain(x, w, b, rng)
        exact = sum(Fraction(float(a)) * Fraction(float(c)) for a, c in zip(x, w)) + Fraction(float(b))
        S = float(sum(abs(Fraction(float(a)) * Fraction(float(c))) for a, c in zip(x, w)) + abs(Fraction(float(b))))
        bnd = X.bound(torch.tensor([S], dtype=torch.float64), X.chain_gamma(3 * K // 16, 1),
                      torch.tensor([float(exact)], dtype=torch.float64)).item()
        err = abs(float(got - exact))
        assert err <= bnd, (K, kind, err, bnd)
        worst = max(worst, err / bnd)
    assert worst > 1e-4                                         # the bound is not vacuous
    print("K=%d %s: worst error %.3f of the bound" % (K, kind, worst))
