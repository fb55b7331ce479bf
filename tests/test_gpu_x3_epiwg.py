"""The two-limb convs drain their accumulators in a dedicated epilogue warpgroup (tc_conv_x3_epiwg_kernel, the default) or in
the MMA warpgroups themselves (tc_conv_x3_kernel, udh_debug_x3_set_epi_wg(0)).  Both sum the same chain of k16 products and
apply the same epilogue arithmetic, so every output bit, ReLU mask word and pool routing code must agree.  Checked for every
instance the train step launches, at the step's shapes (B = 128, 128 x 128 patches), and for one whole train step."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as O                                               # noqa: E402

P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
B = 128


@pytest.fixture(scope="module")
def udh():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from unsuperviseddeephomographyral2018_b200 import _lib, engine, params
    _lib.require_device()

    class NS:
        pass
    ns = NS()
    ns.engine, ns.params, ns.L = engine, params, _lib.lib
    return ns


def _both(udh, run):
    """run() under the epilogue-warpgroup kernel and under the in-warpgroup one; the switch is restored afterwards"""
    res = {}
    try:
        for on in (1, 0):
            assert udh.L.udh_debug_x3_set_epi_wg(on) == 0
            res[on] = run()
            torch.cuda.synchronize()
    finally:
        udh.L.udh_debug_x3_set_epi_wg(1)
    return res[1], res[0]


def _same_bits(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    assert torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)), \
        "%s: %d elements differ" % (what, int((a.view(torch.int32) != b.view(torch.int32)).sum()))


# (H, cin, cout) of conv2_x, conv3_1, conv3_2 and conv4_x; forward (bias + ReLU + ReLU-mask out) and dgrad (ReLU mask in)
@pytest.mark.parametrize("H,cin,cout", [(64, 64, 64), (32, 64, 128), (32, 128, 128), (16, 128, 128)])
@pytest.mark.parametrize("dgrad", [0, 1])
def test_x3_epiwg_generic_instances_bit_identical(udh, H, cin, cout, dgrad):
    g = torch.Generator(device="cuda").manual_seed(H * 7 + cin + cout + dgrad)
    kin, kout = (cout, cin) if dgrad else (cin, cout)
    x = torch.randn(B, H, H, kin, device="cuda", generator=g)
    w = torch.randn(3, 3, cin, cout, device="cuda", generator=g) * 0.05
    bias = None if dgrad else torch.randn(kout, device="cuda", generator=g)
    words = B * (H + 2) * (H + 2) * kout // 32
    mask_in = torch.randint(-2 ** 31, 2 ** 31 - 1, (words,), device="cuda", generator=g, dtype=torch.int32) if dgrad else None
    scratch = torch.empty(udh.L.udh_debug_x3_scratch_bytes(B, H, H, cin, cout), device="cuda", dtype=torch.uint8)

    def run():
        out = torch.full((B, H, H, kout), float("nan"), device="cuda")
        mask_out = None if dgrad else torch.full((words,), -1, device="cuda", dtype=torch.int32)
        assert udh.L.udh_debug_x3_conv_ex(P(x), P(w), P(bias), P(mask_in), P(mask_out), P(out), P(scratch), B, H, H, cin, cout,
                                          0 if dgrad else 1, dgrad, None) == 0, udh.L.udh_last_error()
        return out, mask_out

    (o1, m1), (o0, m0) = _both(udh, run)
    assert not torch.isnan(o1).any()
    _same_bits(o1, o0, "output")
    if not dgrad:
        assert (m1 != -1).any()
        _same_bits(m1, m0, "ReLU mask words")


@pytest.mark.parametrize("rows", [1, 2])
def test_x3_epiwg_conv1_2_row_tiles_bit_identical(udh, rows):
    """conv1_2 on row tiles: rows = 1 forward fused with pool1 (pooled stream + routing codes), rows = 2 dgrad with the mask"""
    H = 128
    g = torch.Generator(device="cuda").manual_seed(40 + rows)
    x = torch.randn(B, H, H, 64, device="cuda", generator=g)
    w = torch.randn(3, 3, 64, 64, device="cuda", generator=g) * 0.05
    bias = torch.randn(64, device="cuda", generator=g) if rows == 1 else None
    words = B * (H + 2) * (H + 2) * 2
    mask_in = torch.randint(-2 ** 31, 2 ** 31 - 1, (words,), device="cuda", generator=g, dtype=torch.int32) if rows == 2 else None
    scratch = torch.empty(udh.L.udh_debug_x3_scratch_bytes(B, H, H, 64, 64), device="cuda", dtype=torch.uint8)
    oh = H // 2 if rows == 1 else H

    def run():
        out = torch.full((B, oh, oh, 64), float("nan"), device="cuda")
        codes = torch.full((B, H // 2, H // 2, 8), -1, device="cuda", dtype=torch.int32) if rows == 1 else None
        assert udh.L.udh_debug_x3_conv_rows(P(x), P(w), P(bias), P(mask_in), P(out), P(codes), P(scratch), B, H, H, rows, None) == 0, \
            udh.L.udh_last_error()
        return out, codes

    (o1, c1), (o0, c0) = _both(udh, run)
    assert not torch.isnan(o1).any()
    _same_bits(o1, o0, "pooled output" if rows == 1 else "dgrad output")
    if rows == 1:
        assert (c1 != -1).all()
        _same_bits(c1, c0, "routing codes")


def test_x3_epiwg_train_step_bit_identical(udh):
    """one forward + backward of the certified step at B = 128: predictions and every gradient bit for bit"""
    seed = 2
    flat = udh.params.init_flat_large(seed)
    db = {k: (v.cuda().contiguous() if isinstance(v, torch.Tensor) else v) for k, v in O.make_batch(seed, B).items()}

    def run():
        e = udh.engine.HomographyEngine(B, seed=None, numeric="bf16x3", loss_type="h_loss", lr=5e-4)
        e.load_flat(flat)
        out = e.forward(db, train=True, dropout_seed=5)
        e.backward(db, out)
        return out["pred_h4p"].clone(), e.grads.clone()

    (p1, g1), (p0, g0) = _both(udh, run)
    assert np.isfinite(g1.cpu().numpy()).all()
    _same_bits(p1, p0, "pred_h4p")
    _same_bits(g1, g0, "gradients")
