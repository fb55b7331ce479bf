"""CPU tests of oracle/optim.py: the float32 schedule of the reference's TF graph, and the per-element error bound of the
Adam kernel checked against exact Fraction arithmetic over every contraction the compiler may choose.  Also pins how the
engine's float64 alpha_t relates to TF's float32 one (DESIGN section 2, "row O and the loop")."""
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import optim as Q

f32 = np.float32
CLI = (1e-4, 0.9e-4)            # homography_CNN_synthetic.py defaults
BENCH = (5e-4, 0.9e-4)          # bench.py


def test_decay_steps_of_both_settings():
    assert Q.decay_steps(*CLI) == 58117 and Q.decay_steps(*BENCH) == 3570


@pytest.mark.parametrize("lr,min_lr", [CLI, BENCH])
def test_staircase_boundaries_fp32(lr, min_lr):
    """The rate steps down exactly at k * decay_steps, never at k * decay_steps - 1, for every k up to step 150 000."""
    ds = Q.decay_steps(lr, min_lr)
    for k in range(0, 150000 // ds + 1):
        want = f32(f32(lr) * f32(float(f32(0.96)) ** k))
        if k > 0:
            assert Q.exponential_decay_fp32(lr, k * ds - 1, ds) == f32(f32(lr) * f32(float(f32(0.96)) ** (k - 1)))
        assert Q.exponential_decay_fp32(lr, k * ds, ds) == want
    assert Q.exponential_decay_fp32(lr, 149999, ds) == f32(f32(lr) * f32(float(f32(0.96)) ** (149999 // ds)))


def test_beta_power_chain():
    """beta_power is multiplied once per update in float32: at t = 3 it is fl(fl(0.9f * 0.9f) * 0.9f), not fp32(0.9^3)."""
    b = f32(0.9)
    assert Q.beta_power_fp32(0.9, 1) == b and Q.beta_power_fp32(0.9, 3) == f32(f32(b * b) * b)
    assert Q.beta_power_fp32(0.9, 3) != f32(0.9 ** 3)
    assert Q.beta_power_fp32(0.999, 150001) == 0 and Q.beta_power_fp32(0.9, 1000) == 0


def _alphas(lr, min_lr, steps):
    """(TF float32 alpha_t, engine alpha_t rounded to the kernel's float32) for global steps `steps`, vectorised."""
    from unsuperviseddeephomographyral2018_b200 import engine
    ds = Q.decay_steps(lr, min_lr)
    t = steps + 1
    Q.beta_power_fp32(0.9, int(t.max())); Q.beta_power_fp32(0.999, int(t.max()))
    p1 = np.array([Q.beta_power_fp32(0.9, int(k)) for k in t], f32)
    p2 = np.array([Q.beta_power_fp32(0.999, int(k)) for k in t], f32)
    lr_t = np.array([Q.exponential_decay_fp32(lr, int(s), ds) for s in np.unique(steps // ds * ds)], f32)[
        np.searchsorted(np.unique(steps // ds * ds), steps // ds * ds)]
    tf = (lr_t * np.sqrt(f32(1) - p2)) / (f32(1) - p1)
    eng = np.array([f32(engine.adam_alpha(int(s), lr, min_lr)[1]) for s in steps], f32)
    return tf.astype(np.float64), eng.astype(np.float64)


def test_tf_alpha_restatement_matches_scalar_form():
    for s in (0, 1, 2, 9, 3569, 3570, 149999):
        lr_t, a = Q.tf_alpha(s, *BENCH)
        tf, _ = _alphas(*BENCH, np.array([s]))
        assert a == f32(tf[0]) and lr_t == Q.exponential_decay_fp32(5e-4, s, 3570)


@pytest.mark.parametrize("lr,min_lr", [CLI, BENCH])
def test_engine_alpha_against_tf_fp32_chain(lr, min_lr):
    """The engine evaluates alpha_t in float64 with exact beta powers; TF in float32 from its beta-power chain.  Decision
    (DESIGN section 2): keep the float64 form.  Over all 150 000 steps of both settings the two differ by <= 1.4e-5 relative,
    worst at t = 3; 6.7e-6 at t = 1, 3.8e-6 at t = 1000, and only lr_t's float32 arithmetic once both beta powers are below
    2^-25."""
    steps = np.arange(0, 150000)
    tf, eng = _alphas(lr, min_lr, steps)
    rel = np.abs(eng - tf) / tf
    worst = int(np.argmax(rel))
    print("lr %g: engine alpha_t vs TF float32 alpha_t: worst %.3e at t = %d" % (lr, rel[worst], worst + 1))
    assert rel.max() <= 1.4e-5 and worst + 1 == 3
    if lr == CLI[0]:
        assert rel[0] == pytest.approx(6.67e-6, rel=1e-2) and rel[2] == pytest.approx(1.36e-5, rel=1e-2)
        assert 3.7e-6 <= abs(eng[999] - tf[999]) / eng[999] <= 3.8e-6
    # at t = 150 000 the bias correction is exactly 1 in both forms; what is left is lr_t, whose float32 base 0.96f carries
    # its rounding into the power (k = 42 at bench.py's setting: 1e-6)
    assert Q.adam_lr_t_fp32(1.0, 150000) == 1.0 and rel[-1] <= 1.2e-6


def test_checkpoint_beta_powers_give_tf_alpha_within_the_bound():
    """The checkpoint writes float32(beta^(t+1)), not the chain's value.  A TF run resumed from it forms its lr_t from those
    powers: that lr_t stays within 1.6e-5 of the chain's (measured 1.53e-5, at the first update after step 1)."""
    from unsuperviseddeephomographyral2018_b200 import params as P, tf_checkpoint as tfc
    specs = P.param_specs()
    n = P.total_floats(specs)
    z = np.zeros(n, f32)
    for step in (0, 1, 2, 9, 999, 3569, 3570, 87292, 149999):
        var = tfc.engine_state_to_variables(z, z, z, step, specs)
        p1, p2 = f32(var["beta1_power"]), f32(var["beta2_power"])
        assert p1 == f32(0.9 ** (step + 1)) and p2 == f32(0.999 ** (step + 1))
        resumed = f32(np.sqrt(f32(1) - p2) / (f32(1) - p1))              # lr_t / lr of the first update after the restore
        chain = Q.adam_lr_t_fp32(1.0, step + 1)
        assert abs(float(resumed) - float(chain)) <= 1.6e-5 * float(chain), step


# ---------------------------------------------------------------------------------------------------- the Adam bound
@pytest.mark.parametrize("gs", [1.0, 0.5, 0.125, 1.0 / 3.0])
def test_adam_bound_holds_against_exact_arithmetic(gs):
    """For 800 inputs per grad_scale, every contraction of the kernel's float32 sequence stays inside adam_bound around the
    exact (Fraction) update; g = m = v = 0 leaves p bit for bit; adam64 agrees with the exact update to float64 rounding."""
    rng = np.random.default_rng(int(gs * 1000))
    n = 800
    p, g, m, v = Q.adam_inputs(rng, n)
    alphas = [f32(Q.tf_alpha(s, *BENCH)[1]) for s in (0, 1, 9, 3569, 149999)]
    worst = {"p": 0.0, "m": 0.0, "v": 0.0}
    for ai, a in enumerate(alphas):
        sl = slice(ai * n // len(alphas), (ai + 1) * n // len(alphas))
        args = (p[sl], g[sl], m[sl], v[sl], a)
        ep, em, ev = Q.adam_bound(*args, grad_scale=gs)
        P64, M64, V64 = Q.adam64(*args, grad_scale=gs)
        exact = [Q.adam_exact(p[sl][i], g[sl][i], m[sl][i], v[sl][i], a, grad_scale=gs) for i in range(len(ep))]
        for i, (Pe, Me, Ve) in enumerate(exact):
            assert abs(Fraction(P64[i]) - Pe) <= 1e-15 * (abs(Pe) + 1e-30) + ep[i] * 1e-6
        for name, pv, mv, vv in Q.adam_fp32_variants(*args, grad_scale=gs):
            for i, (Pe, Me, Ve) in enumerate(exact):
                for key, got, ref, b in (("p", pv[i], Pe, ep[i]), ("m", mv[i], Me, em[i]), ("v", vv[i], Ve, ev[i])):
                    r = float(abs(Fraction(float(got)) - ref)) / b
                    assert r <= 1.0, (name, key, i, float(got), float(ref), b)
                    worst[key] = max(worst[key], r)
            zero = (g[sl] == 0) & (m[sl] == 0) & (v[sl] == 0)
            assert np.array_equal(pv[zero], p[sl][zero])
    print("gs = %.4g: worst measured / bound over all contractions: p %.3f  m %.3f  v %.3f" % (gs, worst["p"], worst["m"], worst["v"]))
    assert worst["p"] > 0.01 and worst["v"] > 0.01       # the bound is not vacuous


def test_adam_bound_separates_eps_conventions():
    """Where sqrt(v) < eps the bound is far tighter than the change an eps inside the sqrt, or the Kingma eps-hat, would make."""
    g = np.array([1e-9, 3e-8, -2e-7], f32)
    z = np.zeros(3, f32)
    p = np.full(3, 1e-2, f32)                                  # a conv weight's magnitude
    a = f32(Q.tf_alpha(0, *BENCH)[1])
    P64, M, V = Q.adam64(p, g, z, z, a)
    ep, _, _ = Q.adam_bound(p, g, z, z, a)
    inside = p - a * M / np.sqrt(V + 1e-8)
    kingma = p - a * M / (np.sqrt(V) + 1e-8 * math.sqrt(1 - 0.999))
    assert np.all(np.abs(inside - P64) > 100 * ep) and np.all(np.abs(kingma - P64) > 100 * ep)
