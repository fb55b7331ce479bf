"""CPU tests of oracle/simt_fp32.py, the restatement of the fp32 CUDA-core engine's arithmetic that
tests/test_gpu_fp32_certify.py holds the kernels to bit for bit: the conv / dgrad chains and the weight-gradient partials
against exact rational evaluation of the same operation order, the any-order bound on the atomics' sum, and the pooling
rule on hand-built tie windows."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import simt_fp32 as S

f32 = np.float32


def round_f32(q):
    """Fraction -> nearest fp32 (ties to even), exactly (no detour through fp64)."""
    if q == 0:
        return f32(0)
    a = abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    quantum = Fraction(2) ** (max(e, -126) - 23)
    r = round(a / quantum) * quantum                         # Fraction.__round__ rounds half to even
    return f32(float(r) if q > 0 else -float(r))


def exact_fma_chain(a, b, start=Fraction(0)):
    acc = start
    for x, y in zip(a, b):
        acc = Fraction(float(round_f32(Fraction(float(x)) * Fraction(float(y)) + acc)))
    return f32(acc)


def _conv_case(seed, B, H, W, cin, cout, dgrad, scale=1.0):
    rng = np.random.default_rng(seed)
    kin = cout if dgrad else cin
    x = (rng.standard_normal((B, H, W, kin)) * scale).astype(f32)
    w = (rng.standard_normal((3, 3, cin, cout)) * 0.3).astype(f32)
    return x, w


def test_round_f32_matches_numpy_on_fp64_values():
    rng = np.random.default_rng(0)
    for v in np.concatenate([rng.standard_normal(500), rng.standard_normal(100) * 1e-40, [1 + 2.0 ** -24, 1 + 3 * 2.0 ** -24]]):
        assert round_f32(Fraction(float(v))) == f32(v), v      # a single rounding from fp64 is correct


@pytest.mark.parametrize("dgrad", [0, 1])
def test_conv_chain_equals_exact_evaluation_of_the_kernel_order(dgrad):
    """Every output of a tiny layer: conv_chain == the same fmaf order evaluated exactly, then + bias, ReLU, mask."""
    B, H, W, cin, cout = 2, 3, 4, 3, 2
    x, w = _conv_case(7 + dgrad, B, H, W, cin, cout, dgrad)
    bias = None if dgrad else np.array([0.3, -0.7], f32)
    kout = cin if dgrad else cout
    mask = np.random.default_rng(3).standard_normal((B, H, W, kout)).astype(f32)
    n, y, xx, o = (a.reshape(-1) for a in np.meshgrid(np.arange(B), np.arange(H), np.arange(W), np.arange(kout), indexing="ij"))
    got = S.conv_chain(x, w, n, y, xx, o, bias=bias, relu=not dgrad, mask=mask, dgrad=bool(dgrad))
    wk = w[::-1, ::-1].transpose(0, 1, 3, 2) if dgrad else w
    for i in range(len(n)):
        a, b = [], []
        for c in range(wk.shape[2]):                      # channel, then ky, kx: the kernel's order
            for ky in range(3):
                for kx in range(3):
                    yy, xc = y[i] + ky - 1, xx[i] + kx - 1
                    a.append(x[n[i], yy, xc, c] if 0 <= yy < H and 0 <= xc < W else f32(0))
                    b.append(wk[ky, kx, c, o[i]])
        v = exact_fma_chain(a, b)
        if bias is not None:
            v = f32(v + bias[o[i]])
        if not dgrad:
            v = max(v, f32(0))
        if not mask[n[i], y[i], xx[i], o[i]] > 0:
            v = f32(0)
        assert got[i] == v, (i, got[i], v)


def test_conv_chain_two_planes_equals_stacked_channels():
    rng = np.random.default_rng(5)
    I1, I2 = (rng.standard_normal((2, 8, 16, 1)).astype(f32) for _ in range(2))
    w = rng.standard_normal((3, 3, 2, 64)).astype(f32)
    n, y, xx, o = rng.integers(0, 2, 50), rng.integers(0, 8, 50), rng.integers(0, 16, 50), rng.integers(0, 64, 50)
    a = S.conv_chain(I1, w, n, y, xx, o, x2=I2)
    b = S.conv_chain(np.concatenate([I1, I2], axis=3), w, n, y, xx, o)
    assert np.array_equal(a, b)


def test_conv_chain_sees_a_change_of_rounding_order():
    """Starting the chain from the bias, or rounding the product before the add, changes the result on some elements: the
    restatement pins the order, not just the value."""
    x, w = _conv_case(11, 1, 8, 16, 64, 64, 0)
    bias = np.random.default_rng(2).standard_normal(64).astype(f32)
    rng = np.random.default_rng(4)
    n, y, xx, o = np.zeros(400, int), rng.integers(0, 8, 400), rng.integers(0, 16, 400), rng.integers(0, 64, 400)
    ref = S.conv_chain(x, w, n, y, xx, o, bias=bias)
    a, b = S.conv_operands(x, w, n, y, xx, o)
    from_bias, unfused = bias[o].copy(), np.zeros(len(o), f32)
    for k in range(a.shape[1]):
        from_bias = S.fmaf32(a[:, k], b[:, k], from_bias)
        unfused = (unfused + (a[:, k] * b[:, k]).astype(f32)).astype(f32)
    unfused = (unfused + bias[o]).astype(f32)
    assert (from_bias != ref).mean() > 0.05 and (unfused != ref).mean() > 0.05
    assert np.abs(from_bias.astype(np.float64) - ref).max() < 1e-4 * np.abs(ref).max()   # rounding-level differences


@pytest.mark.parametrize("two_plane", [False, True])
def test_wgrad_partials_equal_exact_chains_and_cover_every_pixel_once(two_plane):
    B, H, W = 3, 16, 32                                    # 12 tiles
    cin, cout = (2, 64) if two_plane else (16, 64)
    part = (5, 3, 8) if two_plane else (4, 3, 1)           # the last CTA of the first one walks a short range
    rng = np.random.default_rng(9)
    x = rng.standard_normal((B, H, W, cin)).astype(f32)
    g = rng.standard_normal((B, H, W, cout)).astype(f32)
    x1, x2 = (x[..., :1], x[..., 1:]) if two_plane else (x, None)
    ky, kx, ci, co = np.array([0, 1, 2, 2]), np.array([2, 1, 0, 2]), np.array([0, 1, 1, 0]), np.array([5, 63, 0, 17])
    p = S.wgrad_partials(x1, g, part, ky, kx, ci, co, x2=x2)
    pb = S.bias_partials(g, part, co)
    assert p.shape == (4, part[0] * part[2]) and pb.shape == p.shape
    nn, yy, xx, ok = S._partial_terms(B, H, W, part)
    pix = (nn * H + yy) * W + xx
    assert np.array_equal(np.sort(pix[ok]), np.arange(B * H * W))      # every pixel in exactly one partial
    for e in range(4):
        for j in range(p.shape[1]):
            sel = ok[j]
            a = [x[nn[j, t], yy[j, t] + ky[e] - 1, xx[j, t] + kx[e] - 1, ci[e]]
                 if 0 <= yy[j, t] + ky[e] - 1 < H and 0 <= xx[j, t] + kx[e] - 1 < W else f32(0) for t in np.nonzero(sel)[0]]
            b = [g[nn[j, t], yy[j, t], xx[j, t], co[e]] for t in np.nonzero(sel)[0]]
            assert p[e, j] == exact_fma_chain(a, b), (e, j)
            acc = f32(0)
            for v in b:
                acc = f32(acc + v)
            assert pb[e, j] == acc, (e, j)
    # the float64 sum of the partials is the exact dW up to the partials' own rounding
    s, bound = S.sum_bound(p)
    x64 = np.pad(x.astype(np.float64), ((0, 0), (1, 1), (1, 1), (0, 0)))
    for e in range(4):
        ref = (x64[:, ky[e]:ky[e] + H, kx[e]:kx[e] + W, ci[e]] * g[..., co[e]]).sum()
        assert abs(s[e] - ref) <= S.gamma(B * H * W) * np.abs(x64[:, ky[e]:ky[e] + H, kx[e]:kx[e] + W, ci[e]] * g[..., co[e]]).sum()
    assert (bound > 0).all()


def test_sum_bound_holds_for_every_order_of_fp32_atomics():
    rng = np.random.default_rng(1)
    p = (rng.standard_normal(40) * np.exp(rng.uniform(-6, 6, 40))).astype(f32)
    s, bound = S.sum_bound(p)
    worst = 0.0
    for _ in range(300):
        acc = f32(0)
        for v in rng.permutation(p):
            acc = f32(acc + v)
        worst = max(worst, abs(float(acc) - float(Fraction(0) + sum(Fraction(float(v)) for v in p))))
    assert worst <= bound and worst > 0


def _win(vals):
    """One 2x2 window [a b; c d] as an NHWC tensor [1,2,2,1]."""
    return torch.tensor(vals, dtype=torch.float32).reshape(1, 2, 2, 1)


@pytest.mark.parametrize("vals,winner", [
    ([1.0, 3.0, 3.0, 2.0], 1),        # two equal maxima: the first in row-major order
    ([3.0, 3.0, 3.0, 1.0], 0),        # three
    ([2.5, 2.5, 2.5, 2.5], 0),        # four
    ([1.0, 0.5, 4.0, 4.0], 2),        # tie in the second row
    ([-1.0, 2.0, -3.0, 2.0], 1),
    ([0.0, 0.0, 0.0, 0.0], None),     # maximum 0: no gradient
    ([-0.0, 0.0, -0.0, 0.0], None),   # +-0: not > 0
    ([-2.0, -1.0, -5.0, -1.0], None),  # negative maximum (not post-ReLU, but the rule is the same)
    ([2.0 ** -149, 0.0, 0.0, 2.0 ** -149], 0),   # the smallest positive subnormal is > 0
])
def test_pool_rule_on_tie_windows(vals, winner):
    x = _win(vals)
    g = torch.tensor([[[[-7.25]]]])
    assert S.pool_fwd(x).item() == max(vals)
    din = S.pool_bwd(x, g).flatten()
    want = torch.zeros(4)
    if winner is not None:
        want[winner] = -7.25
    assert torch.equal(din.view(torch.int32), want.view(torch.int32)), (din, want)    # bit for bit: +0 elsewhere


def test_pool_rule_on_many_windows_and_channels():
    rng = np.random.default_rng(3)
    x = torch.tensor(rng.integers(-1, 3, size=(2, 6, 8, 4)).astype(np.float32))
    g = torch.tensor(rng.standard_normal((2, 3, 4, 4)).astype(np.float32))
    din = S.pool_bwd(x, g)
    for n in range(2):
        for oy in range(3):
            for ox in range(4):
                for c in range(4):
                    win = [x[n, 2 * oy + dy, 2 * ox + dx, c].item() for dy in (0, 1) for dx in (0, 1)]
                    k = int(np.argmax(win))                    # numpy argmax: first maximum
                    for i, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
                        v = din[n, 2 * oy + dy, 2 * ox + dx, c].item()
                        assert v == (g[n, oy, ox, c].item() if (i == k and max(win) > 0) else 0.0)
    assert torch.equal(S.pool_fwd(x), torch.nn.functional.max_pool2d(x.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1))
