"""Restatement of the two-limb tensor-core mode's number format (UDH_NUMERIC_BF16X3) — TEST INFRASTRUCTURE ONLY.

  * split / join: an fp32 value travels as hi = bf16_rn(x), lo = bf16_rn(x - hi) (round to nearest even, as the kernels'
    __floats2bfloat162_rn), and is read back as the fp32 sum hi + lo.  join(split(x)) keeps the value of x to 2^-16 but the
    split of a joined value is not always the original pair: when x - hi rounds to exactly half an ulp of an odd hi, the
    re-split rounds the tie to the even neighbour of hi and takes the negative half ulp as lo (same value, other limbs).
  * stored(acc, mode): what a conv kernel stores for an fp32 accumulator — join(split(acc)) in the two-limb mode, bf16_rn(acc)
    in the single-pass bf16 mode.
  * every product is hi_x.hi_w + hi_x.lo_w + lo_x.hi_w (three MMA passes, lo.lo dropped by design; conv1_1's weight gradient
    is the exception, it adds all four): `three_pass` gives the exact value of that sum for operands whose limbs are known.
  * exact operand classes: integers (lo = 0) and limb operands (integer hi, lo = k 2^-10 below half an ulp of hi).  Products
    of bf16 values are exact; when every partial sum, in any order and grouping, is a multiple of the grid below 2^22 grid
    units, fp32 accumulation is exact whatever alignment or truncation the tensor core applies internally, provided it keeps
    >= 23 bits — the internal accumulator width of H100 wgmma for bf16 is not documented, so the margin is kept.
    `abs_terms` gives sum |hh| + |hl| + |lh| of every output, and `require_exact` asserts the precondition from it before a
    test launches anything.
  * `bound`: a per-element bound of |kernel - float64| for one output on real data, from the split residuals (2^-16 per
    operand), the dropped lo.lo term, fp32 accumulation over the instance's chain modelled as truncating (u = 2^-23, any
    order), the bias add and the final split of a stored output.
Arrays are torch tensors on any device."""
import torch

from .simt_fp32 import gamma

GRID_LO = 2.0 ** -10          # grid of the limb operands' lo limbs
EXACT_UNITS = 2.0 ** 22       # partial sums below this many grid units are exact with >= 23 accumulator bits
U_ACC = 2.0 ** -23            # fp32 accumulation, truncating
U_BF16 = 2.0 ** -8            # unit roundoff of a bf16 limb (8 significant bits, round to nearest)
# |x w - (hh + hl + lh)| <= C_PROD |x w|: each operand's split residual |x - hi - lo| <= u^2 |x|, |hi + lo| <= (1 + u^2) |x|,
# and the dropped |lo_x lo_w| <= u^2 (1 + u)^2 |x w|
C_PROD = (U_BF16 ** 2) * ((1 + U_BF16) ** 2 + 2 * (1 + U_BF16 ** 2) + U_BF16 ** 2)
# sum of |hh| + |hl| + |lh| <= C_TERMS |x w|
C_TERMS = (1 + U_BF16) ** 2 * (1 + 2 * U_BF16)
# |join(split(v)) - v| <= U_STORE |v|: the split residual plus the rounding of the fp32 sum hi + lo
U_STORE = U_BF16 ** 2 + 2.0 ** -24


def bf16_rn(x):
    return x.float().to(torch.bfloat16).float()


def split(x):
    """(hi, lo) fp32 tensors holding the two bf16 limbs of fp32 x."""
    x = x.float()
    hi = bf16_rn(x)
    return hi, bf16_rn(x - hi)


def join(hi, lo):
    return hi + lo                          # one fp32 add, as tc::join2


def stored(acc, mode="bf16x3"):
    """The value a conv kernel stores for fp32 accumulators acc (read back as fp32)."""
    acc = acc.float()
    if mode == "bf16x3":
        return join(*split(acc))
    if mode == "bf16":
        return bf16_rn(acc)
    raise ValueError(mode)


def three_pass(f, x, w):
    """sum(hh + hl + lh) of a bilinear f (float64 conv / GEMM) on operands whose split is exact: f(x, w) - f(lo_x, lo_w)."""
    lo_x, lo_w = split(x)[1], split(w)[1]
    return f(x.double(), w.double()) - f(lo_x.double(), lo_w.double())


def int_operand(gen, shape, vmax=2, density=1.0, device="cuda"):
    """Integers in [-vmax, vmax] (lo = 0); a fraction 1 - density of them forced to zero."""
    x = torch.randint(-vmax, vmax + 1, shape, device=device, generator=gen).float()
    if density < 1.0:
        x = torch.where(torch.rand(shape, device=device, generator=gen) < density, x, torch.zeros_like(x))
    return x.contiguous()


def limb_operand(gen, shape, with_lo=True, vmax=2, density=1.0, device="cuda"):
    """hi in {+-1 .. +-vmax} (zero with probability 1 - density), lo = k 2^-10 with k in {-1, 0, 1} where hi != 0 (lo = 0
    everywhere when not with_lo).  |lo| <= 2^-10 is below half the ulp of bf16 on either side of every integer 1 .. 2^8, so
    split(hi + lo) returns these limbs: asserted."""
    mag = torch.randint(1, vmax + 1, shape, device=device, generator=gen).float()
    sign = torch.where(torch.rand(shape, device=device, generator=gen) < 0.5, -1.0, 1.0)
    hi = mag * sign
    if density < 1.0:
        hi = torch.where(torch.rand(shape, device=device, generator=gen) < density, hi, torch.zeros_like(hi))
    lo = torch.zeros_like(hi)
    if with_lo:
        lo = torch.randint(-1, 2, shape, device=device, generator=gen).float() * GRID_LO
        lo = torch.where(hi != 0, lo, torch.zeros_like(lo))
    x = (hi + lo).contiguous()
    h2, l2 = split(x)
    assert torch.equal(h2, hi) and torch.equal(l2, lo), "limb operand does not split into its own limbs"
    return x


def abs_terms(f, x, w):
    """sum |hh| + |hl| + |lh| of every output of a bilinear f (float64 conv / GEMM): f(|hi_x|, |hi_w| + |lo_w|) +
    f(|lo_x|, |hi_w|).  (f(|x|, |w|) can understate it by 2 2^-10 relative where lo and hi have opposite signs.)"""
    hx, lx = (t.double().abs() for t in split(x))
    hw, lw = (t.double().abs() for t in split(w))
    return f(hx, hw + lw) + f(lx, hw)


def require_exact(terms, grid, what):
    """Assert the exactness precondition: the sum of |terms| of every output (float64: `abs_terms`, plus |bias| where a
    bias is added) stays below 2^22 grid units, so that every partial sum does."""
    worst = float(terms.max()) / grid
    assert worst < EXACT_UNITS, "%s: sum |terms| reaches %.3g grid units >= 2^22: not exact in fp32" % (what, worst)
    return worst


def chain_gamma(ksteps, extra=0):
    """gamma of the roundings an element's term can see: up to 16 inside one k16 wgmma (order and alignment unspecified),
    one per later accumulating k-step, plus `extra` adds outside the MMA (bias, slab reduction)."""
    return float(gamma(ksteps + 16 + extra, U_ACC))


def bound(abs_xw, g, ref=None):
    """Per-element bound of |kernel - float64| for outputs with sum |x w| (+ |bias|) = abs_xw (float64) and chain gamma g:
    the products' split / lo.lo error, the accumulation over C_TERMS abs_xw, and, when ref (the float64 value) is given, the
    final split of the stored output."""
    e = C_PROD * abs_xw + g * C_TERMS * abs_xw
    if ref is not None:
        e = e + U_STORE * (ref.abs() + e)
    return e
