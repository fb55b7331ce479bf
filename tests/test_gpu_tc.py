"""GPU tests of the tensor-core (UDH_NUMERIC_BF16) path: each wgmma kernel against a torch
reference on bf16-rounded operands (so the only difference is fp32 summation order: tolerance 1e-4 relative to the
largest output), and the whole bf16 engine against the fp32 engine / the oracle.

The single-pass bf16 mode is the THROUGHPUT mode and is NOT parity-certified: on the large-output weights
(params.init_flat_large, |pred_h4p| tens of px) its pred_h4p is within ~1e-2 relative (tenths of a pixel) of fp32 — two to
three orders of magnitude outside the 1e-3 px of BASELINE's north_star; these tests bound and PRINT that error.  The
parity-certified tensor-core mode is UDH_NUMERIC_BF16X3 (tests/test_gpu_x3.py).  Whole-network GRADIENTS cannot agree tightly between bf16 and fp32
arithmetic: a bf16 perturbation of a pre-activation that sits within rounding of zero flips its ReLU (and max-pool
arg-max), which switches that unit's whole gradient path on or off.  Measured on this test: relative L2 difference
0.7 % at fc2, 7 % at fc1, growing to 23 % at conv1_1, cosine similarity 0.97-0.9999 — so the end-to-end check is a
direction check (cosine >= 0.9 per tensor, norm ratio within 15 %), and exactness of the backward kernels is established
layer by layer above (each wgmma kernel vs torch on identical bf16 operands)."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import oracle as O                                               # noqa: E402


@pytest.fixture(scope="module")
def udh():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from unsuperviseddeephomographyral2018_b200 import _lib, engine, ops, params
    _lib.require_device()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False

    class NS:
        pass
    ns = NS()
    ns.lib, ns.ops, ns.engine, ns.params, ns.L = _lib, ops, engine, params, _lib.lib
    return ns


P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None


CONV_CASES = [(2, 128, 64, 64), (3, 64, 64, 64), (2, 32, 64, 128), (2, 32, 128, 128), (5, 16, 128, 128), (1, 16, 128, 128)]


@pytest.mark.parametrize("B,H,cin,cout", CONV_CASES)
@pytest.mark.parametrize("dgrad", [0, 1])
def test_tc_conv_layer(udh, B, H, cin, cout, dgrad):
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + H)
    kin, kout = (cout, cin) if dgrad else (cin, cout)
    x = torch.randn(B, H, H, kin, device="cuda", generator=g).bfloat16().float().contiguous()
    w = (torch.randn(3, 3, cin, cout, device="cuda", generator=g) * 0.05).bfloat16().float().contiguous()
    bias = None if dgrad else torch.randn(kout, device="cuda", generator=g).contiguous()
    out = torch.full((B, H, H, kout), float("nan"), device="cuda")
    scratch = torch.empty(udh.L.udh_debug_tc_conv_scratch_bytes(B, H, H, cin, cout), device="cuda", dtype=torch.uint8)
    assert udh.L.udh_debug_tc_conv(P(x), P(w), P(bias), P(out), P(scratch), B, H, H, cin, cout, 0 if dgrad else 1, dgrad, None) == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    wk = torch.flip(w, dims=(0, 1)).permute(2, 3, 0, 1) if dgrad else w.permute(3, 2, 0, 1)
    ref = F.conv2d(x.permute(0, 3, 1, 2), wk.contiguous(), bias, padding=1)
    ref = (ref if dgrad else F.relu(ref)).permute(0, 2, 3, 1)
    assert (out - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()


@pytest.mark.parametrize("B,H,cin,cout", CONV_CASES)
def test_tc_wgrad_layer(udh, B, H, cin, cout):
    g = torch.Generator(device="cuda").manual_seed(B * 77 + H)
    x = torch.randn(B, H, H, cin, device="cuda", generator=g).bfloat16().float().contiguous()
    go = (torch.randn(B, H, H, cout, device="cuda", generator=g) * 0.1).bfloat16().float().contiguous()
    dW = torch.zeros(3, 3, cin, cout, device="cuda"); db = torch.zeros(cout, device="cuda")
    scratch = torch.empty(udh.L.udh_debug_tc_conv_scratch_bytes(B, H, H, cin, cout), device="cuda", dtype=torch.uint8)
    assert udh.L.udh_debug_tc_wgrad(P(x), P(go), P(dW), P(db), P(scratch), B, H, H, cin, cout, None) == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    ref = torch.nn.grad.conv2d_weight(x.permute(0, 3, 1, 2), (cout, cin, 3, 3), go.permute(0, 3, 1, 2), padding=1).permute(2, 3, 1, 0)
    refb = go.sum(dim=(0, 1, 2))
    assert (dW - ref).abs().max().item() <= 2e-4 * ref.abs().max().item()
    assert (db - refb).abs().max().item() <= 2e-4 * refb.abs().max().item() + 1e-5


def dev(batch):
    return {k: (v.cuda().contiguous() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}


def rel_l2(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)


@pytest.mark.parametrize("loss_type", ["h_loss", "l1_loss"])
def test_bf16_engine_vs_fp32_engine(udh, loss_type):
    seed, B = 0, 4
    batch = dev(O.make_batch(seed, B))
    flat = udh.params.init_flat_large(seed)
    e32 = udh.engine.HomographyEngine(B, seed=None, numeric="fp32", loss_type=loss_type, lr=5e-4); e32.load_flat(flat)
    e16 = udh.engine.HomographyEngine(B, seed=None, numeric="bf16", loss_type=loss_type, lr=5e-4); e16.load_flat(flat)
    o32 = e32.forward(batch, train=True, dropout_seed=123)
    o16 = e16.forward(batch, train=True, dropout_seed=123)
    m32, m16 = e32.dropout_masks(), e16.dropout_masks()
    assert torch.equal(m32[1], m16[1])                                    # same seed -> same fc1 mask
    h32, h16 = o32["pred_h4p"].cpu().numpy(), o16["pred_h4p"].cpu().numpy()
    print("bf16 vs fp32 engine: max|pred| %.1f px, max err %.3f px" % (np.abs(h32).max(), np.abs(h16 - h32).max()))
    assert np.abs(h32).max() > 10.0 and np.abs(h16 - h32).max() <= 3e-2 * np.abs(h32).max()
    e32.backward(batch, o32); e16.backward(batch, o16)
    specs = udh.params.param_specs()
    g32, g16 = e32.grads.cpu(), e16.grads.cpu()
    for name, s in specs.items():
        a, b = g16[s.offset:s.offset + s.size].double(), g32[s.offset:s.offset + s.size].double()
        cos = float(a @ b / (a.norm() * b.norm() + 1e-300))
        assert cos >= 0.9, (name, cos)
        assert 0.85 <= float(a.norm() / b.norm()) <= 1.15, (name, float(a.norm() / b.norm()))
    s2 = specs["model/fc2/fc2/weights"]
    if loss_type == "h_loss":
        assert rel_l2(g16[s2.offset:s2.offset + s2.size], g32[s2.offset:s2.offset + s2.size]) < 6e-2
    d32, d16 = e32.losses_dict(o32), e16.losses_dict(o16)
    assert abs(d32["h_loss"] - d16["h_loss"]) <= 0.5 and abs(d32["l1_loss"] - d16["l1_loss"]) <= 2e-2
    e16.update()
    # cleared for the next step, except fc1's weight gradient: its bf16 GEMM stores rather than accumulates (udh.h)
    s1 = specs["model/fc1/fc1/weights"]
    assert e16.grads[:s1.offset].abs().max().item() == 0.0 and e16.grads[s1.offset + s1.size:].abs().max().item() == 0.0
    assert e16.global_step == 1


def test_bf16_measured_error_on_large_output_golden(udh, golden_dir):
    """What single-pass bf16 costs on a network whose outputs are tens of pixels (NOT a parity claim)."""
    g = np.load(os.path.join(golden_dir, "e2e_golden.npz"))
    for seed in (0, 1):
        eng = udh.engine.HomographyEngine(2, seed=None, numeric="bf16"); eng.load_flat(udh.params.init_flat_large(seed))
        db = dev(O.make_batch(seed, 2))
        db["gt"] = torch.tensor(g["s%d_gt_metric" % seed]).cuda()
        out = eng.forward(db, train=False)
        d = eng.losses_dict(out)
        ps = np.abs(g["s%d_pred_h4p" % seed]).max()
        e = np.abs(out["pred_h4p"].cpu().numpy() - g["s%d_pred_h4p" % seed]).max()
        dm = abs(d["bounded_h_loss"] - float(g["s%d_bounded_h_loss_m" % seed]))
        print("bf16 single pass, seed %d: max|pred| %.1f px, max err %.3f px (%.2e relative), |d mean corner error| %.3f px" % (seed, ps, e, e / ps, dm))
        assert e <= 5e-2 * ps and dm <= 0.5


def test_bf16_full_size_properties_B128(udh):
    """BASELINE configs[1] size (B = 128) in the tensor-core mode: replicated samples agree with the B = 4 run (the tiling
    of the padded streams must not leak between images), the mean corner error agrees with the fp32 mode to 1e-3 px, and a
    train step leaves finite, non-trivial updates in every parameter tensor."""
    B = 128
    batch = O.make_batch(100, 4)
    flat = udh.params.init_flat_large(0)
    rep = lambda t: t.repeat(B // 4, *([1] * (t.dim() - 1))).cuda().contiguous()
    db = {k: rep(v) for k, v in batch.items() if isinstance(v, torch.Tensor) and k != "H_gt"}
    e16 = udh.engine.HomographyEngine(B, seed=None, numeric="bf16", loss_type="h_loss", lr=5e-4); e16.load_flat(flat)
    out = e16.forward(db, train=False)
    h = out["pred_h4p"].clone()
    hs = h.abs().max().item()
    assert hs > 10.0
    assert (h[:4] - h[4:8]).abs().max().item() < 2e-6 * hs and (h[:4] - h[-4:]).abs().max().item() < 2e-6 * hs
    e4 = udh.engine.HomographyEngine(4, seed=None, numeric="bf16"); e4.load_flat(flat)
    h4 = e4.forward(dev(batch), train=False)["pred_h4p"]
    assert (h4 - h[:4]).abs().max().item() < 2e-6 * hs
    e32 = udh.engine.HomographyEngine(B, seed=None, numeric="fp32"); e32.load_flat(flat)
    d32, d16 = e32.losses_dict(e32.forward(db, train=False)), e16.losses_dict(out)
    # throughput mode: tenths of a pixel, not 1e-3 px (the certified tensor-core mode is bf16x3)
    assert abs(d32["bounded_h_loss"] - d16["bounded_h_loss"]) <= 0.5 and abs(d32["h_loss"] - d16["h_loss"]) <= 0.5
    del e32
    p0 = e16.params.clone()
    e16.train_step(db)
    specs = udh.params.param_specs()
    upd = (e16.params - p0)
    assert torch.isfinite(e16.params).all()
    for name, s in specs.items():
        u = upd[s.offset:s.offset + s.size]
        assert u.abs().max().item() > 0, name                     # every tensor received a gradient
        assert u.abs().max().item() <= 5e-4 * 1.01, name          # first TF-Adam step is bounded by lr


def test_adam_refreshes_fc1_mirror(udh):
    """bf16 mode: Adam writes the bf16 copy of fc1's weights in the same pass (udh_adam_step_mirror) and the next forward
    skips its own conversion.  The mirror must equal round-to-nearest bf16 of the updated fp32 weights bit for bit, the
    gradient of that range is left in place (its GEMM stores), every other gradient is cleared, and a forward that trusts
    the mirror equals one that re-derives it."""
    B = 4
    db = dev(O.make_batch(7, B))
    eng = udh.engine.HomographyEngine(B, seed=0, numeric="bf16", loss_type="h_loss", lr=5e-4)
    assert eng._mirror is not None
    mp, mb, mc, stored = eng._mirror
    assert stored == 1
    s = eng.specs["model/fc1/fc1/weights"]
    assert (mb, mc) == (s.offset, s.size)
    for _ in range(2):
        eng.train_step(db)
    assert eng._mirror_current
    off = mp - eng.ws.data_ptr()
    mirror = eng.ws[off:off + 2 * mc].view(torch.bfloat16)
    want = eng.params[mb:mb + mc].to(torch.bfloat16)
    assert torch.equal(mirror.view(torch.int16), want.view(torch.int16))
    g = eng.grads
    assert g[:mb].abs().max().item() == 0 and g[mb + mc:].abs().max().item() == 0 and g[mb:mb + mc].abs().max().item() > 0
    a = eng.eval_step(db)["pred_h4p"].clone()                      # uses the mirror
    eng._mirror_current = False
    b = eng.eval_step(db)["pred_h4p"].clone()                      # converts again
    assert (a - b).abs().max().item() <= 1e-5 * max(1.0, b.abs().max().item())
    # a torch in-place write to the parameters invalidates the mirror by itself (version counter), a C-side update does not
    eng.train_step(db)
    assert eng._mirror_is_current()
    eng.params.mul_(1.0)
    assert not eng._mirror_is_current()
    c = eng.eval_step(db)["pred_h4p"].clone()
    assert torch.isfinite(c).all()
    fp = udh.engine.HomographyEngine(B, seed=0, numeric="fp32")
    assert fp._mirror is None


@pytest.mark.parametrize("B,H", [(1, 4), (3, 128)])
def test_tc_conv_pool_fused(udh, B, H):
    """conv1_2 + pool1 in one kernel (row-pair tiles, 2x2 maximum in the epilogue) against torch on the same bf16-rounded
    operands: pooled activations, and routing codes that must point at an element equal to the window maximum (4 exactly
    where the maximum is not positive)."""
    W = 128
    g = torch.Generator(device="cuda").manual_seed(B * 31 + H)
    x = torch.randn(B, H, W, 64, device="cuda", generator=g).bfloat16().float().contiguous()
    w = (torch.randn(3, 3, 64, 64, device="cuda", generator=g) * 0.06).bfloat16().float().contiguous()
    bias = (torch.randn(64, device="cuda", generator=g) * 0.1).contiguous()
    pooled = torch.empty(B, H // 2, W // 2, 64, device="cuda")
    codes = torch.zeros(B, H // 2, W // 2, 8, device="cuda", dtype=torch.int32)
    scratch = torch.empty(udh.L.udh_debug_tc_conv_scratch_bytes(B, H, W, 64, 64), device="cuda", dtype=torch.uint8)
    assert udh.L.udh_debug_tc_conv_pool(P(x), P(w), P(bias), P(pooled), P(codes), P(scratch), B, H, W, None) == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    full = torch.relu(torch.nn.functional.conv2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), bias, padding=1))   # [B,64,H,W]
    ref = torch.nn.functional.max_pool2d(full, 2).permute(0, 2, 3, 1)
    tol = 1e-2 * ref.abs().max().item()
    assert (pooled - ref).abs().max().item() <= tol
    # decode the codes: channel c of pooled pixel -> 3 bits at (c % 8) * 3 of word c // 8
    sh = (torch.arange(64, device="cuda") % 8) * 3
    k = (codes.long()[..., torch.arange(64, device="cuda") // 8] >> sh) & 7                  # [B,H/2,W/2,64]
    assert int(k.max()) <= 4
    win = full.permute(0, 2, 3, 1).reshape(B, H // 2, 2, W // 2, 2, 64).permute(0, 1, 3, 5, 2, 4).reshape(B, H // 2, W // 2, 64, 4)
    picked = torch.gather(win, 4, k.clamp(max=3).unsqueeze(-1)).squeeze(-1)
    live = k < 4
    assert (picked[live] - ref[live]).abs().max().item() <= tol
    assert ref[~live].abs().max().item() <= tol if (~live).any() else True
    assert (ref[live] > -tol).all()
    assert live.float().mean().item() > 0.5
