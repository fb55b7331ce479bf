"""Row O in TF's own arithmetic and in float64, with the per-element error bound of the Adam kernel.

* The schedule as the reference graph evaluates it (code/homography_CNN_synthetic.py:161-183): `tf.train.exponential_decay`
  with staircase=True, and `AdamOptimizer`'s lr_t, both in float32 as TF 1.x computes them:
    - exponential_decay casts global_step, decay_steps and decay_rate to the learning rate's dtype (float32) and returns
      lr * pow(decay_rate, floor(global_step / decay_steps));
    - AdamOptimizer keeps two float32 variables beta1_power / beta2_power, created at beta1 / beta2 and multiplied by the
      float32 beta once after every update; ApplyAdam forms lr_t = lr * sqrt(1 - beta2_power) / (1 - beta1_power) in float32.
  TF's kernels run with subnormals flushed to zero, so the chain ends at 0 instead of stalling at a subnormal; lr_t is the
  same either way, since 1 - beta_power rounds to 1 long before the chain leaves the normal range.
* `adam64`: the update of libudh's adam_kernel (csrc/misc.cu) in float64 from the kernel's own float32 inputs.
* `adam_bound`: a bound on |kernel - adam64| per element, from the kernel's operation sequence with u = 2^-24.
"""
import math
from fractions import Fraction

import numpy as np

f32 = np.float32
U = 2.0 ** -24
TINY = 2.0 ** -140          # absolute slack for results that pass through the subnormal range


# ---------------------------------------------------------------------------------------------------- the schedule
def decay_steps(lr, min_lr, num_total_steps=150000, decay_rate=0.96):
    """int(decay_steps) of homography_CNN_synthetic.py:166,169 (Python floats, as the script computes it)."""
    return int((math.log(decay_rate) * num_total_steps) / math.log(min_lr * 1.0 / lr))


def exponential_decay_fp32(lr, step, ds, decay_rate=0.96):
    """tf.train.exponential_decay(lr, step, ds, decay_rate, staircase=True) in float32.  pow is taken as correctly rounded
    (the float64 power of the float32 base, rounded once)."""
    p = np.floor(f32(step) / f32(ds))
    return f32(f32(lr) * f32(float(f32(decay_rate)) ** float(p)))


_CHAIN = {}


def beta_power_fp32(beta, k):
    """AdamOptimizer's float32 beta-power variable before update k (1-based): beta at k = 1, times beta once per update."""
    c = _CHAIN.setdefault(float(f32(beta)), [f32(beta)])
    b = f32(beta)
    while len(c) < k:
        x = f32(c[-1] * b)
        c.append(x if abs(x) >= np.finfo(f32).tiny else f32(0))
    return c[k - 1]


def adam_lr_t_fp32(lr_t, t, beta1=0.9, beta2=0.999):
    """ApplyAdam's float32 lr_t = lr * sqrt(1 - beta2_power) / (1 - beta1_power) at update t (1-based)."""
    one = f32(1)
    p1, p2 = beta_power_fp32(beta1, t), beta_power_fp32(beta2, t)
    return f32(f32(f32(lr_t) * np.sqrt(f32(one - p2))) / f32(one - p1))


def tf_alpha(step, lr, min_lr):
    """(lr_t, alpha_t) of the update that moves global_step from `step` to step + 1, in TF's float32 arithmetic."""
    lr_t = exponential_decay_fp32(lr, step, decay_steps(lr, min_lr))
    return lr_t, adam_lr_t_fp32(lr_t, step + 1)


# ---------------------------------------------------------------------------------------------------- Adam in float64
# adam64 / adam_bound take float32 NumPy arrays or float32 torch tensors (CPU or CUDA) and answer in float64 of the same kind.
def _ops(x):
    if isinstance(x, np.ndarray) or np.isscalar(x):
        return (lambda t: np.asarray(t, f32).astype(np.float64)), (lambda t, gs: (np.asarray(t, f32) * f32(gs)).astype(np.float64)), np
    import torch
    return (lambda t: t.float().double()), (lambda t, gs: (t.float() * float(f32(gs))).double()), torch


def _consts(alpha, beta1, beta2, eps, grad_scale):
    b1, b2, e, a, gs = (float(f32(x)) for x in (beta1, beta2, eps, alpha, grad_scale))
    return b1, b2, e, a, gs, float(f32(1) - f32(beta1)), float(f32(1) - f32(beta2))


def adam64(p, g, m, v, alpha, beta1=0.9, beta2=0.999, eps=1e-8, grad_scale=1.0):
    """adam_kernel's update in float64 on its float32 inputs: returns (p', m', v').  1 - beta is exact in float32 (Sterbenz),
    so c1, c2 are the kernel's own constants."""
    d, _, xp = _ops(p)
    b1, b2, e, a, gs, c1, c2 = _consts(alpha, beta1, beta2, eps, grad_scale)
    G = d(g) * gs
    M = b1 * d(m) + c1 * G
    V = b2 * d(v) + c2 * G * G
    return d(p) - a * M / (xp.sqrt(V) + e), M, V


def adam_bound(p, g, m, v, alpha, beta1=0.9, beta2=0.999, eps=1e-8, grad_scale=1.0):
    """Per-element bounds (ep, em, ev) on |kernel - adam64| for p', m', v'.

    adam_kernel computes, in float32: g' = g*gs; m' = b1*m + c1*g'; v' = b2*v + c2*g'*g'; p' = p - alpha*m' / (sqrt(v') + eps).
      g'  = g*gs rounded once (exact for a power-of-two gs); its error is carried exactly below, g' being known;
      m'  <= 2u (|b1 m| + |c1 g'|) around b1 m + c1 g' (two roundings, or one product and one FMA: m' can cancel, so the
          bound is on the operands, not on m');
      v'  <= 3u (b2 v + c2 g'^2) (all terms are >= 0);
      s   = sqrt(v') + eps: the propagated v' error, then u for the sqrt and u for the sum;
      q   = alpha*m' / s: u for the product and u for the quotient, plus the propagated m' and s errors;
      p'  = p - q: u |p'|.
    An FMA rounds once where the separate operations round twice, so contraction only lowers each term: the one bound holds
    for any choice ptxas makes.  gamma_k = k u / (1 - k u) absorbs the second-order terms."""
    d, gprime, xp = _ops(p)
    gam = lambda k: k * U / (1 - k * U)
    b1, b2, e, a, gs, c1, c2 = _consts(alpha, beta1, beta2, eps, grad_scale)
    G = d(g) * gs
    gp = gprime(g, gs)                                                     # the kernel's g'
    M = b1 * d(m) + c1 * G
    V = b2 * d(v) + c2 * G * G
    em = gam(2) * (xp.abs(b1 * d(m)) + xp.abs(c1 * gp)) * (1 + 4 * U) + c1 * xp.abs(gp - G) + TINY
    ev = gam(3) * (b2 * d(v) + c2 * gp * gp) * (1 + 4 * U) + c2 * xp.abs(gp * gp - G * G) * (1 + 4 * U) + TINY
    S = xp.sqrt(V) + e
    if xp is np:
        with np.errstate(divide="ignore"):
            dsq = np.minimum(np.sqrt(ev), ev / np.sqrt(V))                 # |sqrt(a) - sqrt(b)| <= min(sqrt|a-b|, |a-b|/sqrt(b))
    else:
        dsq = xp.minimum(xp.sqrt(ev), ev / xp.sqrt(V))
    es = dsq + gam(2) * (xp.sqrt(V + ev) + e) * (1 + 4 * U)
    s_lo = S - es
    s_lo = s_lo * (s_lo > e * 0.5) + (e * 0.5) * (s_lo <= e * 0.5)
    aM = xp.abs(M)
    eq = (gam(2) * a * (aM + em) / s_lo + a * (em / s_lo + aM * es / (s_lo * S))) * (1 + 4 * U) + TINY
    P = d(p) - a * M / S
    ep = eq + gam(1) * (xp.abs(P) + eq) * (1 + 4 * U) + TINY
    return ep, em, ev


def adam_inputs(rng, n):
    """float32 (p, g, m, v) across the regimes where the update goes wrong: |g| in {0, 1e-12, 1e-9, 3e-7, 1e-4, 1, 1e3} with
    mixed signs; t = 1 (m = v = 0); steady state (v ~ g^2); sqrt(v) ~ eps; m opposite to g; g = m = v = 0."""
    mag = np.array([0, 1e-12, 1e-9, 3e-7, 1e-4, 1.0, 1e3])
    g = mag[rng.integers(0, len(mag), n)] * rng.uniform(0.5, 2.0, n) * rng.choice([-1, 1], n)
    kind = rng.integers(0, 5, n)
    m = np.where(kind == 0, 0, np.where(kind == 3, -g * rng.uniform(0.1, 2, n), g * rng.uniform(-1, 1, n)))
    v = np.where(kind == 0, 0, np.where(kind == 2, (1e-8 * rng.uniform(0.3, 3, n)) ** 2, g * g * rng.uniform(0.5, 2, n)))
    z = kind == 4
    g, m, v = np.where(z, 0, g), np.where(z, 0, m), np.where(z, 0, v)
    p = rng.normal(size=n) * 10.0 ** rng.integers(-4, 2, n)
    return [np.asarray(x, f32) for x in (p, g, m, v)]


# ---------------------------------------------------------------------------------------------------- exact arithmetic
def _sqrt_fraction(x, bits=160):
    """sqrt of a non-negative Fraction to within 2^-bits relative (floor of the scaled integer root)."""
    if x == 0:
        return Fraction(0)
    k = bits - (x.numerator.bit_length() - x.denominator.bit_length()) // 2
    r = math.isqrt(x.numerator * 4 ** k // x.denominator)
    return Fraction(r, 2 ** k)


def adam_exact(p, g, m, v, alpha, beta1=0.9, beta2=0.999, eps=1e-8, grad_scale=1.0):
    """The same update as adam64 on scalars, in Fraction arithmetic (sqrt to 2^-160): the yardstick adam_bound is tested on."""
    F = lambda x: Fraction(float(f32(x)))
    b1, b2, e, a, gs = F(beta1), F(beta2), F(eps), F(alpha), F(grad_scale)
    c1, c2 = 1 - b1, 1 - b2
    G = F(g) * gs
    M = b1 * F(m) + c1 * G
    V = b2 * F(v) + c2 * G * G
    return F(p) - a * M / (_sqrt_fraction(V) + e), M, V


def adam_fp32_variants(p, g, m, v, alpha, beta1=0.9, beta2=0.999, eps=1e-8, grad_scale=1.0):
    """adam_kernel's float32 arithmetic in every contraction ptxas may choose (arrays): yields (name, p', m', v').
    m' = b1*m + c1*g': separate, fma(b1, m, c1*g'), fma(c1, g', b1*m); v' = b2*v + (c2*g')*g': separate,
    fma(c2*g', g', b2*v), fma(b2, v, (c2*g')*g').  sqrt and the division are IEEE (nvcc's default -prec-sqrt / -prec-div)."""
    from oracle.warp_fp32 import fmaf32
    A = lambda x: np.asarray(x, f32)
    p, g, m, v = A(p), A(g), A(m), A(v)
    b1, b2, e, a, gs = (f32(x) for x in (beta1, beta2, eps, alpha, grad_scale))
    c1, c2 = f32(1) - b1, f32(1) - b2
    gp = g * gs
    ms = dict(sep=(b1 * m) + (c1 * gp), fma_m=fmaf32(b1, m, c1 * gp), fma_g=fmaf32(c1, gp, b1 * m))
    c2g = c2 * gp
    vs = dict(sep=(b2 * v) + (c2g * gp), fma_g=fmaf32(c2g, gp, b2 * v), fma_v=fmaf32(b2, v, c2g * gp))
    for mk, mm in ms.items():
        for vk, vv in vs.items():
            s = np.sqrt(vv) + e
            yield "m:%s v:%s" % (mk, vk), p - (a * mm) / s, mm, vv
