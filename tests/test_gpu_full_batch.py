"""GPU tests of the tensor-core kernels and the train step at the batch sizes the step actually runs.

The persistent kernels give each CTA the items blockIdx.x + i * gridDim.x.  At the B <= 5 shapes of test_gpu_x3.py /
test_gpu_tc.py a CTA gets at most two items; at the B = 128 of the timed train step it walks up to 62 of them (conv1_2's row
tiles), and the split-K weight gradients spread their slabs over every SM.  Everything here runs at that scale:
  * every layer kernel (two-limb and single-pass bf16; forward with and without ReLU, dgrad, wgrad, conv1_1) at B = 1, at a
    ragged B whose two-tile items end half empty, and at B = 128, against float64 torch on the GPU, checked per image;
  * conv1_2's row-tile kernels (forward fused with pool1 + routing codes, dgrad with conv1_1's mask fused) and the fused
    ReLU-mask epilogues (mask_bits in, mask_out out) through udh_debug_x3_conv_rows / udh_debug_x3_conv_ex;
  * grid shapes: udh_set_sm_reserve(n) for n in {0, 1, 7, 64, 127} (forward / dgrad bit-identical across n, weight
    gradients within tolerance at every n and bit-identical on repeat);
  * the whole two-limb step at B = 128 on 128 distinct samples: activations, fc1, the backward on fixed gates (B = 128, 129),
    end-to-end gradients, row tiles vs the unfused path, run-to-run determinism, the data-parallel SM knobs on one GPU;
  * the warp + photometric losses at B = 128 / 512 and the one-call step at B = 128.
Each test prints its measured error next to the bound it asserts."""
import ctypes

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


def dev(batch):
    return {k: (v.cuda().contiguous() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}


def rel_l2(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).norm() / max(b.norm().item(), 1e-30)).item()


# ------------------------------------------------------------------------------------------------ shapes
# the conv instances the step launches: (name, spatial size, cin, cout); conv2_1 and conv2_2 share one instance, and so do
# conv4_1 and conv4_2.  conv1_2 runs on row tiles by default; its generic kernels are the unfused path.
LAYERS = [("conv1_2", 128, 64, 64), ("conv2_x", 64, 64, 64), ("conv3_1", 32, 64, 128), ("conv3_2", 32, 128, 128),
          ("conv4_x", 16, 128, 128)]


def tiles_per_item(cin, cout, dgrad):
    """T of the launcher's instance (conv_x3.cu tc_conv_x3): two 128-row tiles per item when the output has 64 channels."""
    kout = cin if dgrad else cout
    return 2 if kout == 64 else 1


def num_tiles(B, H):
    return -(-B * (H + 2) * (H + 2) // 128)


# A batch size whose last item is half empty in every two-tile instance the step launches (conv1_2 and conv2_x forward /
# dgrad at 128 and 64 px, conv3_1's dgrad at 32 px): an odd tile count there.
RAGGED_B = 70
BATCHES = [1, RAGGED_B, 128]


def test_ragged_batch_ends_in_a_half_empty_item():
    for H in (128, 64, 32):
        assert num_tiles(RAGGED_B, H) % 2 == 1, H
    assert num_tiles(128, 128) % 2 == 0                   # B = 128 itself fills its last item


def _check_images(got, ref, tol, what, T=None):
    """max |got - ref| <= tol * max |ref| over the tensor AND per image (against that image's own max |ref|); the failure
    message names the image, the position and, for conv outputs, the 128-row tile / item of the padded stream."""
    got, ref = got.double(), ref.double()
    scale = ref.abs().max().item()
    assert scale > 0, what
    d = (got - ref).abs()
    err = d.max().item() / scale
    per = d.flatten(1).max(dim=1)
    img_scale = ref.abs().flatten(1).max(dim=1).values.clamp_min(1e-300)
    rel = per.values / img_scale
    bad = (rel > tol).nonzero().flatten().tolist()
    msgs = []
    for n in bad[:4]:
        idx = per.indices[n].item()
        pos = np.unravel_index(idx, tuple(ref.shape[1:]))
        m = "image %d at %s (rel err %.2e)" % (n, tuple(int(p) for p in pos), rel[n].item())
        if T is not None and ref.dim() == 4:
            Hh, Ww = ref.shape[1], ref.shape[2]
            q = (n * (Hh + 2) + pos[0] + 1) * (Ww + 2) + pos[1] + 1
            m += ", tile %d, item %d" % (q // 128, q // 128 // T)
        msgs.append(m)
    assert err <= tol and not bad, "%s: max rel err %.2e > %.0e; %d images fail: %s" % (what, err, tol, len(bad), "; ".join(msgs))
    return err


def _ref_conv(x, w, bias, relu, dgrad):
    wk = torch.flip(w, dims=(0, 1)).permute(2, 3, 0, 1) if dgrad else w.permute(3, 2, 0, 1)
    r = F.conv2d(x.double().permute(0, 3, 1, 2), wk.double().contiguous(), None if bias is None else bias.double(), padding=1)
    return (F.relu(r) if relu else r).permute(0, 2, 3, 1)


def _ref_wgrad(x, go, cin, cout):
    dW = torch.nn.grad.conv2d_weight(x.double().permute(0, 3, 1, 2), (cout, cin, 3, 3), go.double().permute(0, 3, 1, 2), padding=1)
    return dW.permute(2, 3, 1, 0), go.double().sum(dim=(0, 1, 2))


def _inputs(seed, B, H, kin, cin, cout, bias=True, round_bf16=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, H, H, kin, device="cuda", generator=g)
    w = torch.randn(3, 3, cin, cout, device="cuda", generator=g) * 0.05
    if round_bf16:
        x, w = x.bfloat16().float(), w.bfloat16().float()
    b = torch.randn(cout, device="cuda", generator=g).contiguous() if bias else None
    return x.contiguous(), w.contiguous(), b


# ------------------------------------------------------------------------------------------------ 1. layer kernels vs fp64
def _x3_conv(udh, x, w, bias, B, H, cin, cout, relu, dgrad, mask_bits=None, mask_out=None):
    kout = cin if dgrad else cout
    out = torch.full((B, H, H, kout), float("nan"), device="cuda")
    scratch = torch.empty(udh.L.udh_debug_x3_scratch_bytes(B, H, H, cin, cout), device="cuda", dtype=torch.uint8)
    rc = udh.L.udh_debug_x3_conv_ex(P(x), P(w), P(bias), P(mask_bits), P(mask_out), P(out), P(scratch), B, H, H, cin, cout, relu,
                                    dgrad, None)
    assert rc == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    return out


def _x3_wgrad(udh, x, go, B, H, cin, cout):
    dW = torch.zeros(3, 3, cin, cout, device="cuda"); db = torch.zeros(cout, device="cuda")
    scratch = torch.empty(udh.L.udh_debug_x3_scratch_bytes(B, H, H, cin, cout), device="cuda", dtype=torch.uint8)
    assert udh.L.udh_debug_x3_wgrad(P(x), P(go), P(dW), P(db), P(scratch), B, H, H, cin, cout, None) == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    return dW, db


@pytest.mark.parametrize("mode", ["fwd_relu", "fwd_linear", "dgrad"])
@pytest.mark.parametrize("name,H,cin,cout", LAYERS)
@pytest.mark.parametrize("B", BATCHES)
def test_x3_conv_layer_at_step_batch_vs_fp64(udh, B, name, H, cin, cout, mode):
    dgrad = int(mode == "dgrad")
    relu = int(mode == "fwd_relu")
    kin = cout if dgrad else cin
    x, w, bias = _inputs(B * 1000 + H + 7 * dgrad + relu, B, H, kin, cin, cout, bias=not dgrad)
    out = _x3_conv(udh, x, w, bias, B, H, cin, cout, relu, dgrad)
    T = tiles_per_item(cin, cout, dgrad)
    err = _check_images(out, _ref_conv(x, w, bias, relu, dgrad), 2e-5, "x3 %s %s B=%d" % (name, mode, B), T)
    print("x3 %-8s %-10s B=%3d (%d tiles of T=%d): max rel err %.2e" % (name, mode, B, num_tiles(B, H), T, err))


def wgrad_tol(B):
    """The weight-gradient kernels sum all the items of a CTA in ONE fp32 wgmma register accumulator, so their rounding error
    grows with the products a CTA accumulates: <= 2e-5 at B <= 5 (test_gpu_x3.py) and at B = 1 here, but measured 1.1e-4 for
    conv1_2 (wgrad64, 16 items per CTA) at B = 128 on the full grid (H100 SXM, 700 W).  A summation bug (a lost, doubled or
    stale item) is >= 1/items per CTA, i.e. >= 4e-3 on the full grid."""
    return 2e-5 if B <= 5 else 2e-4


def wgrad_tol_reserved(B, n):
    """wgrad_tol on a grid of (SMs - n) CTAs: the products per CTA, and with them the error, grow like SMs / (SMs - n)
    (measured 3.5e-3 for conv1_2 and up to 8.7e-4 for the others with 127 of 132 SMs reserved)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return wgrad_tol(B) * sms / max(sms - n, 1)


@pytest.mark.parametrize("name,H,cin,cout", LAYERS)
@pytest.mark.parametrize("B", BATCHES)
def test_x3_wgrad_layer_at_step_batch_vs_fp64(udh, B, name, H, cin, cout):
    g = torch.Generator(device="cuda").manual_seed(B * 77 + H)
    x = torch.randn(B, H, H, cin, device="cuda", generator=g).contiguous()
    go = (torch.randn(B, H, H, cout, device="cuda", generator=g) * 0.1).contiguous()
    dW, db = _x3_wgrad(udh, x, go, B, H, cin, cout)
    ref, refb = _ref_wgrad(x, go, cin, cout)
    e1 = (dW.double() - ref).abs().max().item() / ref.abs().max().item()
    e2 = (db.double() - refb).abs().max().item() / refb.abs().max().item()
    print("x3 %-8s wgrad      B=%3d: dW max rel err %.2e, db %.2e" % (name, B, e1, e2))
    assert e1 <= wgrad_tol(B) and e2 <= wgrad_tol(B), (e1, e2)


def _x3_conv1(udh, I1, I2, w, bias, go, B, H):
    out = torch.full((B, H, H, 64), float("nan"), device="cuda") if w is not None else None
    dW = torch.zeros(3, 3, 2, 64, device="cuda"); db = torch.zeros(64, device="cuda")
    scratch = torch.empty(udh.L.udh_debug_x3_scratch_bytes(B, H, H, 64, 64), device="cuda", dtype=torch.uint8)
    rc = udh.L.udh_debug_x3_conv1(P(I1), P(I2), P(w), P(bias), P(out), P(go), P(dW) if go is not None else None,
                                  P(db) if go is not None else None, P(scratch), B, H, H, None)
    assert rc == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    return out, dW, db


@pytest.mark.parametrize("B", BATCHES)
def test_x3_conv1_1_at_step_batch_vs_fp64(udh, B):
    H = 128
    g = torch.Generator(device="cuda").manual_seed(B * 5 + 3)
    I1 = torch.randn(B, H, H, device="cuda", generator=g).contiguous(); I2 = torch.randn(B, H, H, device="cuda", generator=g).contiguous()
    w = (torch.randn(3, 3, 2, 64, device="cuda", generator=g) * 0.2).contiguous()
    bias = (torch.randn(64, device="cuda", generator=g) * 0.1).contiguous()
    go = (torch.randn(B, H, H, 64, device="cuda", generator=g) * 0.1).contiguous()
    out, dW, db = _x3_conv1(udh, I1, I2, w, bias, go, B, H)
    x = torch.stack([I1, I2], dim=1).double()
    ref = F.relu(F.conv2d(x, w.double().permute(3, 2, 0, 1), bias.double(), padding=1)).permute(0, 2, 3, 1)
    e0 = _check_images(out, ref, 2e-5, "x3 conv1_1 fwd B=%d" % B)
    refw = torch.nn.grad.conv2d_weight(x, (64, 2, 3, 3), go.double().permute(0, 3, 1, 2), padding=1).permute(2, 3, 1, 0)
    refb = go.double().sum(dim=(0, 1, 2))
    e1 = (dW.double() - refw).abs().max().item() / refw.abs().max().item()
    e2 = (db.double() - refb).abs().max().item() / refb.abs().max().item()
    print("x3 conv1_1 B=%3d: fwd %.2e, dW %.2e, db %.2e" % (B, e0, e1, e2))
    assert e1 <= wgrad_tol(B) and e2 <= wgrad_tol(B), (e1, e2)


# single-pass bf16 (the throughput mode): the same kernels' tiling on bf16-rounded operands, so the only difference from the
# float64 reference is fp32 accumulation order
@pytest.mark.parametrize("mode", ["fwd_relu", "dgrad", "wgrad"])
@pytest.mark.parametrize("name,H,cin,cout", LAYERS)
@pytest.mark.parametrize("B", BATCHES)
def test_bf16_layer_at_step_batch(udh, B, name, H, cin, cout, mode):
    scratch = torch.empty(udh.L.udh_debug_tc_conv_scratch_bytes(B, H, H, cin, cout), device="cuda", dtype=torch.uint8)
    if mode == "wgrad":
        g = torch.Generator(device="cuda").manual_seed(B * 77 + H)
        x = torch.randn(B, H, H, cin, device="cuda", generator=g).bfloat16().float().contiguous()
        go = (torch.randn(B, H, H, cout, device="cuda", generator=g) * 0.1).bfloat16().float().contiguous()
        dW = torch.zeros(3, 3, cin, cout, device="cuda"); db = torch.zeros(cout, device="cuda")
        assert udh.L.udh_debug_tc_wgrad(P(x), P(go), P(dW), P(db), P(scratch), B, H, H, cin, cout, None) == 0, udh.L.udh_last_error()
        torch.cuda.synchronize()
        ref, refb = _ref_wgrad(x, go, cin, cout)
        e1 = (dW.double() - ref).abs().max().item() / ref.abs().max().item()
        e2 = (db.double() - refb).abs().max().item() / refb.abs().max().item()
        print("bf16 %-8s wgrad    B=%3d: dW %.2e, db %.2e" % (name, B, e1, e2))
        assert e1 <= 2e-4 and e2 <= 2e-4, (e1, e2)
        return
    dgrad = int(mode == "dgrad")
    kin, kout = (cout, cin) if dgrad else (cin, cout)
    x, w, bias = _inputs(B * 1000 + H + dgrad, B, H, kin, cin, cout, bias=not dgrad, round_bf16=True)
    out = torch.full((B, H, H, kout), float("nan"), device="cuda")
    rc = udh.L.udh_debug_tc_conv(P(x), P(w), P(bias), P(out), P(scratch), B, H, H, cin, cout, 1 - dgrad, dgrad, None)
    assert rc == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    err = _check_images(out, _ref_conv(x, w, bias, 1 - dgrad, dgrad), 1e-4, "bf16 %s %s B=%d" % (name, mode, B))
    print("bf16 %-8s %-8s B=%3d: max rel err %.2e" % (name, mode, B, err))


def _decode_codes(codes):
    sh = (torch.arange(64, device="cuda") % 8) * 3
    return (codes.long()[..., torch.arange(64, device="cuda") // 8] >> sh) & 7              # [B,H/2,W/2,64]


def _check_pool_codes(k, full, tol):
    """full: fp64 conv + bias (before ReLU) [B,H,W,64].  A code equals the fp64 arg-max (first maximum in window order) wherever
    the two largest window values differ by more than tol; elsewhere it points at an element within tol of the maximum.  It is
    4 wherever the maximum is below -tol and < 4 wherever it is above tol."""
    B, H, W, C = full.shape
    win = full.reshape(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(B, H // 2, W // 2, C, 4)
    top2 = win.topk(2, dim=-1).values
    mx, gap = top2[..., 0], top2[..., 0] - top2[..., 1]
    kref = win.argmax(dim=-1)
    assert int(k.max()) <= 4
    assert (k[mx < -tol] == 4).all(), "a window whose maximum is negative routes a gradient"
    assert (k[mx > tol] < 4).all(), "a window with a positive maximum routes no gradient"
    live = k < 4
    clear = live & (gap > tol)
    assert torch.equal(k[clear], kref[clear]), "%d routing codes disagree with the fp64 arg-max" % int((k[clear] != kref[clear]).sum())
    picked = torch.gather(win, 4, k.clamp(max=3).unsqueeze(-1)).squeeze(-1)
    assert ((mx - picked)[live] <= tol).all()
    return live.float().mean().item()


@pytest.mark.parametrize("B", BATCHES)
def test_bf16_conv_pool_at_step_batch(udh, B):
    H = W = 128
    g = torch.Generator(device="cuda").manual_seed(B * 31 + 5)
    x = torch.randn(B, H, W, 64, device="cuda", generator=g).bfloat16().float().contiguous()
    w = (torch.randn(3, 3, 64, 64, device="cuda", generator=g) * 0.06).bfloat16().float().contiguous()
    bias = (torch.randn(64, device="cuda", generator=g) * 0.1).contiguous()
    pooled = torch.full((B, H // 2, W // 2, 64), float("nan"), device="cuda")
    codes = torch.full((B, H // 2, W // 2, 8), -1, device="cuda", dtype=torch.int32)
    scratch = torch.empty(udh.L.udh_debug_tc_conv_scratch_bytes(B, H, W, 64, 64), device="cuda", dtype=torch.uint8)
    assert udh.L.udh_debug_tc_conv_pool(P(x), P(w), P(bias), P(pooled), P(codes), P(scratch), B, H, W, None) == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    full = _ref_conv(x, w, bias, 0, 0)
    ref = F.max_pool2d(F.relu(full).permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
    # the pooled stream is bf16: one rounding of the output (2^-8 relative) on top of the 1e-4 of the accumulation
    scale = ref.abs().max().item()
    d = (pooled.double() - ref).abs()
    assert (d <= 2.0 ** -8 * ref.abs() + 1e-4 * scale).all(), d.max().item() / scale
    frac = _check_pool_codes(_decode_codes(codes), full, 1e-4 * scale)
    print("bf16 conv1_2+pool1 B=%3d: max rel err %.2e, live codes %.3f" % (B, d.max().item() / scale, frac))


# ------------------------------------------------------------------------------------------------ 2. row tiles and masks
def _x3_rows(udh, x, w, bias, B, H, rows, mask_bits=None):
    W = 128
    if rows == 1:
        out = torch.full((B, H // 2, W // 2, 64), float("nan"), device="cuda")
        codes = torch.full((B, H // 2, W // 2, 8), -1, device="cuda", dtype=torch.int32)
    else:
        out, codes = torch.full((B, H, W, 64), float("nan"), device="cuda"), None
    scratch = torch.empty(udh.L.udh_debug_x3_scratch_bytes(B, H, W, 64, 64), device="cuda", dtype=torch.uint8)
    rc = udh.L.udh_debug_x3_conv_rows(P(x), P(w), P(bias), P(mask_bits), P(out), P(codes), P(scratch), B, H, W, rows, None)
    assert rc == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    return out, codes


def _random_mask_words(seed, B, H, W, C):
    """uint32 mask words over the padded positions ([B*(H+2)*(W+2), C/32] as int32) and the per-element {0,1} mask they
    encode for the interior [B,H,W,C] (bit j of word k = channel 32k + j)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    words = torch.randint(-2 ** 31, 2 ** 31, (B, H + 2, W + 2, C // 32), device="cuda", generator=g, dtype=torch.int64)
    bits = (words[..., None] >> torch.arange(32, device="cuda")) & 1                       # [B,Hp,Wp,C/32,32]
    m = bits.reshape(B, H + 2, W + 2, C)[:, 1:H + 1, 1:W + 1].double()
    return words.to(torch.int32).contiguous(), m


def _mask_of(out):
    """out > 0 as the kernel's mask words over padded positions (zero words on the border)."""
    B, H, W, C = out.shape
    bits = (out > 0).long().reshape(B, H, W, C // 32, 32) << torch.arange(32, device="cuda")
    words = torch.zeros(B, H + 2, W + 2, C // 32, device="cuda", dtype=torch.int64)
    words[:, 1:H + 1, 1:W + 1] = bits.sum(dim=-1)
    return words.to(torch.int32)            # wraps to the same 32 bits


@pytest.mark.parametrize("B", [1, 3, 128])
def test_x3_rows_conv_pool_and_codes_vs_fp64(udh, B):
    H = 128
    x, w, bias = _inputs(B * 13 + 1, B, H, 64, 64, 64)
    bias = bias * 0.1
    pooled, codes = _x3_rows(udh, x, w, bias, B, H, 1)
    full = _ref_conv(x, w, bias, 0, 0)
    ref = F.max_pool2d(F.relu(full).permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
    err = _check_images(pooled, ref, 2e-5, "x3 conv1_2+pool1 rows B=%d" % B)
    frac = _check_pool_codes(_decode_codes(codes), full, 2e-5 * ref.abs().max().item())
    print("x3 conv1_2+pool1 (row tiles) B=%3d: pooled max rel err %.2e, live codes %.3f" % (B, err, frac))


@pytest.mark.parametrize("B", [1, 3, 128])
def test_x3_rows_dgrad_with_fused_mask_vs_fp64(udh, B):
    H = 128
    g, w, _ = _inputs(B * 17 + 2, B, H, 64, 64, 64, bias=False)
    words, m = _random_mask_words(B + 99, B, H, 128, 64)
    out, _ = _x3_rows(udh, g, w, None, B, H, 2, mask_bits=words)
    ref = _ref_conv(g, w, None, 0, 1)
    err = _check_images(out, ref * m, 2e-5, "x3 conv1_2 dgrad rows + mask B=%d" % B)
    assert (out[m == 0] == 0).all()
    plain, _ = _x3_rows(udh, g, w, None, B, H, 2)
    e2 = _check_images(plain, ref, 2e-5, "x3 conv1_2 dgrad rows B=%d" % B)
    print("x3 conv1_2 dgrad (row tiles) B=%3d: masked %.2e, unmasked %.2e" % (B, err, e2))


# the generic instances whose epilogue fuses a mask in the step: forward of conv2_1 / conv3_1 / conv4_1 writes mask_out, the
# dgrad of conv2_2 / conv3_2 / conv4_2 reads the mask of the layer below
MASK_LAYERS = [("conv2_x", 64, 64, 64), ("conv3_x", 32, 64, 128), ("conv3_2", 32, 128, 128), ("conv4_x", 16, 128, 128)]


@pytest.mark.parametrize("name,H,cin,cout", MASK_LAYERS)
@pytest.mark.parametrize("B", [1, 3, 128])
def test_x3_fused_mask_epilogues(udh, B, name, H, cin, cout):
    # forward: mask_out == (out > 0) bit for bit, including zero words on the border
    x, w, bias = _inputs(B * 23 + H, B, H, cin, cin, cout)
    mo = torch.full((B * (H + 2) * (H + 2), cout // 32), -1, device="cuda", dtype=torch.int32)
    out = _x3_conv(udh, x, w, bias, B, H, cin, cout, 1, 0, mask_out=mo)
    e1 = _check_images(out, _ref_conv(x, w, bias, 1, 0), 2e-5, "x3 %s fwd + mask_out B=%d" % (name, B))
    want = _mask_of(out).reshape(mo.shape)
    assert torch.equal(mo, want), "%d mask words differ from out > 0" % int((mo != want).sum())
    # dgrad: out == fp64 dgrad x mask
    g, w2, _ = _inputs(B * 29 + H, B, H, cout, cin, cout, bias=False)
    words, m = _random_mask_words(B * 31 + H, B, H, H, cin)
    out2 = _x3_conv(udh, g, w2, None, B, H, cin, cout, 0, 1, mask_bits=words)
    e2 = _check_images(out2, _ref_conv(g, w2, None, 0, 1) * m, 2e-5, "x3 %s dgrad + mask B=%d" % (name, B), tiles_per_item(cin, cout, 1))
    assert (out2[m == 0] == 0).all()
    print("x3 %-8s B=%3d: fwd + mask_out %.2e (mask exact), dgrad x mask %.2e" % (name, B, e1, e2))


# ------------------------------------------------------------------------------------------------ 3. grid shapes
RESERVES = [0, 1, 7, 64, 127]


@pytest.fixture
def sm_reserve(udh):
    """set(n) = udh_set_sm_reserve(n); the setting is process-wide, so it is always put back to 0."""
    def set_(n):
        assert udh.L.udh_set_sm_reserve(n) == 0, udh.L.udh_last_error()
    yield set_
    udh.L.udh_set_sm_reserve(0)


FWD_INSTANCES = [(name, H, cin, cout, dgrad) for (name, H, cin, cout) in LAYERS for dgrad in (0, 1)] + \
                [("conv1_2 rows", 128, 64, 64, 1), ("conv1_2 rows", 128, 64, 64, 2)]


@pytest.mark.parametrize("name,H,cin,cout,kind", FWD_INSTANCES)
def test_x3_conv_bit_identical_across_sm_reserve(udh, sm_reserve, name, H, cin, cout, kind):
    """Each item is computed by one CTA in a fixed MMA order, so the output cannot depend on the grid size."""
    B = 128
    rows = name.endswith("rows")
    dgrad = int(kind == 1) if not rows else int(kind == 2)
    kin = cout if dgrad else cin
    x, w, bias = _inputs(4242 + H + kind, B, H, kin, cin, cout, bias=not dgrad)
    words = _random_mask_words(77, B, H, H, 64)[0] if rows and kind == 2 else None
    first = None
    for n in RESERVES:
        sm_reserve(n)
        if rows:
            out, codes = _x3_rows(udh, x, w, bias, B, H, kind, mask_bits=words)
        else:
            out, codes = _x3_conv(udh, x, w, bias, B, H, cin, cout, 1 - dgrad, dgrad), None
        if first is None:
            first = (out, codes)
            continue
        assert torch.equal(out, first[0]), "%s (%s): output with %d SMs reserved differs from the full grid (max %.3g)" % (
            name, "dgrad" if dgrad else "fwd", n, (out - first[0]).abs().max().item())
        if codes is not None:
            assert torch.equal(codes, first[1]), (name, n)
    print("x3 %-12s %-5s B=128: bit-identical for SM reserve %s" % (name, "dgrad" if dgrad else "fwd", RESERVES))


WGRAD_INSTANCES = [("conv1_1", 128, 2, 64)] + [(name, H, cin, cout) for (name, H, cin, cout) in LAYERS]


@pytest.mark.parametrize("name,H,cin,cout", WGRAD_INSTANCES)
def test_x3_wgrad_under_sm_reserve(udh, sm_reserve, name, H, cin, cout):
    """The split-K slab partition follows the grid, so the weight gradient may change in the last bits with n; at every n it
    stays within wgrad_tol_reserved of fp64 and two runs at the same n are bit-identical."""
    B = 128
    g = torch.Generator(device="cuda").manual_seed(H * 3 + cin)
    go = (torch.randn(B, H, H, cout, device="cuda", generator=g) * 0.1).contiguous()
    if name == "conv1_1":
        I1 = torch.randn(B, H, H, device="cuda", generator=g).contiguous(); I2 = torch.randn(B, H, H, device="cuda", generator=g).contiguous()
        x = torch.stack([I1, I2], dim=3)
        run = lambda: _x3_conv1(udh, I1, I2, None, None, go, B, H)[1:]
    else:
        x = torch.randn(B, H, H, cin, device="cuda", generator=g).contiguous()
        run = lambda: _x3_wgrad(udh, x, go, B, H, cin, cout)
    ref, refb = _ref_wgrad(x, go, cin, cout)
    errs = []
    for n in RESERVES:
        sm_reserve(n)
        dW, db = run()
        dW2, db2 = run()
        assert torch.equal(dW, dW2) and torch.equal(db, db2), "%s: two runs with %d SMs reserved differ" % (name, n)
        e1 = (dW.double() - ref).abs().max().item() / ref.abs().max().item()
        e2 = (db.double() - refb).abs().max().item() / refb.abs().max().item()
        errs.append(max(e1, e2))
        assert e1 <= wgrad_tol_reserved(B, n) and e2 <= wgrad_tol_reserved(B, n), (name, n, e1, e2)
    print("x3 %-8s wgrad B=128: max rel err per SM reserve %s = %s" % (name, RESERVES, " ".join("%.2e" % e for e in errs)))


# ------------------------------------------------------------------------------------------------ 4. whole step at B = 128
_BATCHES = {}


def _batch(seed, B):
    if (seed, B) not in _BATCHES:
        _BATCHES[(seed, B)] = O.make_batch(seed, B)
    return _BATCHES[(seed, B)]


@pytest.fixture
def unfused(udh):
    """conv1_2 on the generic kernels + separate pool1 (its full-resolution activation exists); restored afterwards."""
    udh.L.udh_debug_x3_set_rows(0)
    yield
    udh.L.udh_debug_x3_set_rows(1)


ACT_ORDER = {0: "model/conv_block1/conv1", 1: "model/conv_block1/conv2", 8: "pool1", 2: "model/conv_block2/conv1",
             3: "model/conv_block2/conv2", 9: "pool2", 4: "model/conv_block3/conv1", 5: "model/conv_block3/conv2", 10: "pool3",
             6: "model/conv_block4/conv1", 7: "model/conv_block4/conv2"}


def _fp64_params(udh, flat):
    return udh.params.unflatten(torch.tensor(flat).double().cuda(), udh.params.param_specs())


def test_x3_activations_B128_vs_fp64(udh):
    """Every saved activation of the two-limb forward at B = 128 (128 distinct samples) against float64 on the GPU: the unfused
    path for conv1_2, the default row-tile path for pool1, and fc1."""
    seed, B = 3, 128
    flat = udh.params.init_flat_large(seed)
    batch = _batch(seed, B)
    x = torch.cat([batch["I1_aug"], batch["I2_aug"]], dim=3).cuda().double()
    with torch.no_grad():
        _, acts = O.vgg_forward(_fp64_params(udh, flat), x, None, return_acts=True)
    got = {}
    for rows in (0, 1):
        udh.L.udh_debug_x3_set_rows(rows)
        try:
            e3 = udh.engine.HomographyEngine(B, seed=None, numeric="bf16x3"); e3.load_flat(flat)
            e3.forward(dev(batch), train=False)
            layers = list(ACT_ORDER) if rows == 0 else [8]
            for layer in layers:
                got[(rows, layer)] = e3.activation(layer).clone()
            got[(rows, 11)] = e3.activation(11).clone()
            del e3
        finally:
            udh.L.udh_debug_x3_set_rows(1)
    for (rows, layer), a in got.items():
        name = ACT_ORDER.get(layer, "fc1")
        ref = acts[name]
        ref = ref.permute(0, 2, 3, 1).contiguous() if ref.dim() == 4 else ref
        err = _check_images(a.reshape(ref.shape), ref, 3e-5, "%s (%s path)" % (name, "row-tile" if rows else "unfused"))
        print("B=128 %-26s (%s) max rel err %.2e" % (name, "row tiles" if rows else "unfused  ", err))


@pytest.mark.parametrize("B", [1, 128, 129])
def test_x3_fc1_vs_fp64_on_engine_input(udh, B):
    """fc1 alone: relu(conv4_2 . W + b) in float64 from the engine's own conv4_2 output (fc1's input: there is no pool after
    block 4), so only the segment GEMM is measured; B = 129 puts a second, one-row M tile behind a full one."""
    flat = udh.params.init_flat_large(5)
    batch = _batch(5, 128)
    if B != 128:
        idx = torch.arange(B) % 128
        batch = {k: (v[idx] if isinstance(v, torch.Tensor) and v.dim() > 0 and v.shape[0] == 128 else v) for k, v in batch.items()}
    e3 = udh.engine.HomographyEngine(B, seed=None, numeric="bf16x3"); e3.load_flat(flat)
    e3.forward(dev(batch), train=False)
    x = e3.activation(7).reshape(B, -1).double()                  # conv4_2, NHWC flatten (slim.flatten)
    fc1 = e3.activation(11).reshape(B, 1024)
    p = _fp64_params(udh, flat)
    ref = F.relu(x @ p["model/fc1/fc1/weights"] + p["model/fc1/fc1/biases"])
    err = _check_images(fc1, ref, 3e-5, "fc1 B=%d" % B)
    print("fc1 vs fp64 on the engine's conv4_2, B=%3d: max rel err %.2e" % (B, err))


@pytest.mark.parametrize("B", [128, 129])
@pytest.mark.parametrize("loss_type", ["h_loss", "l1_loss"])
def test_x3_backward_equals_fp32_backward_on_same_forward_state_full_batch(udh, loss_type, B, unfused):
    """test_gpu_x3.py's same-gates backward at the step's batch.  B = 129 leaves a K tail of one sample after full k-blocks in
    fc1's weight gradient.  Bound 2e-4 relative L2 per tensor instead of 1e-4: the weight-gradient accumulation of wgrad_tol
    puts conv1_2's weights at 1.1e-4 at B = 128 (every other tensor <= 9e-5)."""
    seed = 0
    flat = udh.params.init_flat_large(seed)
    db = dev(_batch(seed, B))
    e32 = udh.engine.HomographyEngine(B, seed=None, numeric="fp32", loss_type=loss_type, lr=5e-4); e32.load_flat(flat)
    e3 = udh.engine.HomographyEngine(B, seed=None, numeric="bf16x3", loss_type=loss_type, lr=5e-4); e3.load_flat(flat)
    o3 = e3.forward(db, train=True, dropout_seed=123)
    e32.forward(db, train=True, dropout_seed=123)
    n = e3.materialize_activations()
    e32.ws[:n].copy_(e3.ws[:n])
    e3.backward(db, o3)
    e32.backward(db, o3)
    bad, worst = [], 0.0
    for name, s in udh.params.param_specs().items():
        r = rel_l2(e3.grads[s.offset:s.offset + s.size], e32.grads[s.offset:s.offset + s.size])
        worst = max(worst, r)
        if r > 2e-4:
            bad.append((name, r))
    print("%s B=%d: x3 backward vs fp32 backward on the same gates, worst tensor rel L2 %.2e" % (loss_type, B, worst))
    assert not bad, bad


def _fp64_h_loss_grads(udh, flat, batch, keep):
    """d h_loss / d params in float64 on the GPU (h_loss does not depend on the warp, so vgg_forward is the whole oracle)."""
    specs = udh.params.param_specs()
    flat64 = torch.tensor(flat).double().cuda().requires_grad_(True)
    params = {n: flat64[s.offset:s.offset + s.size].reshape(s.shape) for n, s in specs.items()}
    x = torch.cat([batch["I1_aug"], batch["I2_aug"]], dim=3).cuda().double()
    pred = O.vgg_forward(params, x, keep)
    (pred - batch["gt"].cuda().double()).square().mean().sqrt().backward()
    return pred.detach(), flat64.grad


def test_x3_gradients_B128_vs_fp64(udh):
    """End-to-end h_loss gradients at B = 128 against float64 (same dropout masks), at the flip-limited level of
    test_x3_gradients_vs_fp64_oracle, next to the fp32 CUDA-core engine's own distance."""
    seed, B = 0, 128
    flat = udh.params.init_flat_large(seed)
    batch = _batch(seed, B)
    db = dev(batch)
    e32 = udh.engine.HomographyEngine(B, seed=None, numeric="fp32", loss_type="h_loss", lr=5e-4); e32.load_flat(flat)
    e3 = udh.engine.HomographyEngine(B, seed=None, numeric="bf16x3", loss_type="h_loss", lr=5e-4); e3.load_flat(flat)
    o32 = e32.forward(db, train=True, dropout_seed=321); o3 = e3.forward(db, train=True, dropout_seed=321)
    m3 = e3.dropout_masks()
    e32.backward(db, o32); e3.backward(db, o3)
    pred64, g64 = _fp64_h_loss_grads(udh, flat, batch, (m3[0].double(), m3[1].double()))
    scale = pred64.abs().max().item()
    e_pred = (o3["pred_h4p"].double() - pred64).abs().max().item() / scale
    print("B=128 pred_h4p vs fp64 (train mode): x3 %.2e, fp32 engine %.2e" % (e_pred, (o32["pred_h4p"].double() - pred64).abs().max().item() / scale))
    assert e_pred <= 3e-5
    bad = []
    for name, s in udh.params.param_specs().items():
        t = g64[s.offset:s.offset + s.size]
        r3, r32 = rel_l2(e3.grads[s.offset:s.offset + s.size], t), rel_l2(e32.grads[s.offset:s.offset + s.size], t)
        print("B=128 %-34s rel L2 vs fp64: x3 %.2e   fp32 engine %.2e" % (name, r3, r32))
        if r3 > 3e-2:
            bad.append((name, r3, r32))
    assert not bad, bad


def test_x3_rowtile_pool_fusion_equals_unfused_path_B128(udh):
    seed, B = 2, 128
    flat = udh.params.init_flat_large(seed)
    db = dev(_batch(seed, B))
    res = {}
    try:
        for rows in (1, 0):
            udh.L.udh_debug_x3_set_rows(rows)
            e = udh.engine.HomographyEngine(B, seed=None, numeric="bf16x3", loss_type="h_loss", lr=5e-4); e.load_flat(flat)
            out = e.forward(db, train=True, dropout_seed=5)
            pool1 = e.activation(8).clone()
            e.backward(db, out)
            res[rows] = (out["pred_h4p"].clone(), pool1, e.grads.clone())
            del e
    finally:
        udh.L.udh_debug_x3_set_rows(1)
    scale = res[0][0].abs().max().item()
    e_pool = (res[1][1] - res[0][1]).abs().max().item() / res[0][1].abs().max().item()
    e_pred = (res[1][0] - res[0][0]).abs().max().item() / scale
    worst = max(rel_l2(res[1][2][s.offset:s.offset + s.size], res[0][2][s.offset:s.offset + s.size])
                for s in udh.params.param_specs().values())
    print("B=128 row tiles vs unfused: pool1 %.2e, pred_h4p %.2e, worst gradient rel L2 %.2e" % (e_pool, e_pred, worst))
    assert e_pool <= 1e-6 and e_pred <= 2e-6 and worst <= 2e-3


def _step(udh, e, db):
    """HomographyEngine.train_step on one GPU, keeping a copy of the gradient from before the update clears it."""
    a = e._fill_args(db, True)
    e._apply_sm_policy()
    udh.lib.check(udh.L.udh_step_forward_backward(ctypes.byref(a), udh.lib.STEP_ALL, udh.ops._stream()), "udh_step_forward_backward")
    out = e._step_out(db)
    res = dict(grads=e.grads.clone(), pred=out["pred_h4p"].clone(), metrics=out["h4p_metrics"].clone(), photo=out["photo_losses"].clone())
    e.update()
    mp, mb, mc, _ = e._mirror
    off = mp - e.ws.data_ptr()
    limbs = 2 if e.numeric_name == "bf16x3" else 1
    res.update(params=e.params.clone(), m=e.adam_m.clone(), v=e.adam_v.clone(), mirror=e.ws[off:off + 2 * limbs * mc].clone())
    return res


@pytest.mark.parametrize("numeric", ["bf16x3", "bf16"])
def test_train_step_B128_is_deterministic(udh, numeric):
    """Two h_loss steps (the step bench.py times) from identical state give bit-identical gradients, parameters, Adam moments,
    fc1 mirror, predictions and h4p losses.  The photometric losses are fp64 atomic sums (DESIGN section 7): equal to float
    rounding only."""
    B = 128
    flat = udh.params.init_flat_large(4)
    db = dev(_batch(4, B))
    runs = []
    for _ in range(2):
        e = udh.engine.HomographyEngine(B, seed=None, numeric=numeric, loss_type="h_loss", lr=5e-4); e.load_flat(flat)
        e.dropout_seed = 1234
        runs.append(_step(udh, e, db))
        del e
    a, b = runs
    for k in ("grads", "params", "m", "v", "mirror", "pred", "metrics"):
        assert torch.equal(a[k], b[k]), "%s: %s differs between two identical steps" % (numeric, k)
    assert (a["photo"] - b["photo"]).abs().max().item() <= 1e-6 * a["photo"].abs().max().item()
    assert a["grads"].abs().max().item() > 0
    print("%s B=128 h_loss step: bit-identical over two runs" % numeric)


def test_x3_dp_sm_knobs_on_one_gpu(udh):
    """The knobs the data-parallel engine sets (conv4_x reserve 32, backward marker at layer 3 with SMs of its own, a global
    reserve) only move work between SMs: gradients within 1e-5 relative L2 of the default, bit-identical on repeat.  The engine
    applies its _sm_policy at every step, so the policy is set there."""
    B = 128
    flat = udh.params.init_flat_large(6)
    db = dev(_batch(6, B))
    res = []
    try:
        for policy in (None, dict(reserve=8, top=32, marker=3, marker_sms=16), dict(reserve=8, top=32, marker=3, marker_sms=16)):
            e = udh.engine.HomographyEngine(B, seed=None, numeric="bf16x3", loss_type="h_loss", lr=5e-4); e.load_flat(flat)
            e.dropout_seed = 99
            if policy is not None:
                e._sm_policy = policy
            res.append(_step(udh, e, db)["grads"])
            del e
    finally:
        udh.L.udh_set_sm_reserve(0); udh.L.udh_set_sm_reserve_top(0); udh.L.udh_set_bwd_marker(-1); udh.L.udh_set_sm_reserve_marker(0)
    assert torch.equal(res[1], res[2]), "the step under the data-parallel SM policy is not reproducible"
    worst = 0.0
    for name, s in udh.params.param_specs().items():
        r = rel_l2(res[1][s.offset:s.offset + s.size], res[0][s.offset:s.offset + s.size])
        worst = max(worst, r)
        assert r <= 1e-5, (name, r)
    print("B=128 x3 step under the data-parallel SM knobs: worst gradient rel L2 vs default %.2e, bit-identical on repeat" % worst)


# ------------------------------------------------------------------------------------------------ 5. warp, losses, one-call step
def _well_conditioned_batch(seed, B):
    """B samples of make_batch with H = H_gt + noise whose window stays clear of the horizon (where fp32 is undefined, see
    test_gpu_parity._check_pred), so that the batch sums are comparable."""
    batch = O.make_batch(seed, B + B // 4)
    n = B + B // 4
    h4p = batch["gt"] + torch.tensor(np.random.default_rng(seed).normal(0, 2.0, size=(n, 8)).astype(np.float32))
    H = O.solve_dlt(batch["pts1"], h4p)
    pred, cond = O.transform(batch["I_aug"], H, batch["patch_indices"], 128, return_cond=True)
    keep = (cond.flatten(1).max(dim=1).values < 1e2).nonzero().flatten()[:B]
    assert keep.numel() == B
    sub = {k: batch[k][keep] for k in ("I_aug", "I2_aug", "patch_indices")}
    return sub, H[keep], pred[keep], cond[keep]


def _check_pred(pred, ref, cond, frac=0.999, tol=2e-4, mean_tol=2e-5):
    d = (pred.double() - ref.double()).abs()
    t = tol + 1e-6 * cond.double()
    assert (d <= t).double().mean().item() >= frac, "only %.5f of pixels within tolerance (max %g)" % ((d <= t).double().mean().item(), d.max().item())
    assert d.median().item() <= mean_tol and (d / t).mean().item() <= 0.2
    return d.max().item()


@pytest.mark.parametrize("B", [128, 512])
def test_warp_loss_forward_full_batch_vs_oracle(udh, B):
    """At B = 128 / 512 a thread of the warp kernel's grid-stride loop handles several quads.  B = 512 is the B = 128 set four
    times over (same H), so every copy must reproduce the first."""
    sub, H, ref_pred, cond = _well_conditioned_batch(11, 128)
    rep = B // 128
    I_aug, I2 = sub["I_aug"].repeat(rep, 1, 1, 1), sub["I2_aug"].repeat(rep, 1, 1, 1)
    pi, Hr = sub["patch_indices"].repeat(rep, 1), H.repeat(rep, 1, 1)
    ref_pred, cond = ref_pred.repeat(rep, 1, 1, 1), cond.repeat(rep, 1, 1, 1)
    pred, sums = udh.ops.warp_loss_forward(I_aug.cuda().contiguous(), Hr.float().cuda().contiguous(), I2.cuda().contiguous(),
                                           pi.cuda().contiguous(), 128, 128)
    dmax = _check_pred(pred.cpu(), ref_pred, cond)
    pl = udh.ops.photo_losses(pred, I2.cuda().contiguous(), sums, 128, 128, B).cpu().numpy()
    ref = O.losses(None, None, ref_pred.double(), I2.double())
    L = udh.lib
    errs = []
    for name, slot in (("rec_loss", L.L_REC), ("ssim_loss", L.L_SSIM), ("l1_loss", L.L_L1), ("l1_smooth_loss", L.L_L1_SMOOTH),
                       ("ncc_loss", L.L_NCC)):
        r = ref[name].item()
        errs.append(abs(pl[slot] - r) / abs(r))
        assert abs(pl[slot] - r) <= 1e-4 * abs(r) + 1e-6, (name, pl[slot], r)
    p = pred.cpu()
    for k in range(1, rep):
        assert torch.equal(p[k * 128:(k + 1) * 128], p[:128]), "copy %d of the batch differs from the first" % k
    print("warp B=%d: per-pixel max err %.2e, losses max rel err %.2e" % (B, dmax, max(errs)))


@pytest.mark.parametrize("loss_name", ["l1_loss", "ssim_loss"])
def test_warp_loss_backward_B128_vs_fp64_autograd(udh, loss_name):
    B = 128
    batch = O.make_batch(21, B, dtype=torch.float64)
    h4p = batch["gt"] + torch.tensor(np.random.default_rng(3).normal(0, 1.5, size=(B, 8)))
    H = O.solve_dlt(batch["pts1"], h4p).detach()
    # d loss / d H per sample: the loss is a mean over the whole batch, so chunks of it can be differentiated one at a time
    g = torch.zeros_like(H)
    n_total = B * 128 * 128
    for c in range(0, B, 32):
        sl = slice(c, c + 32)
        Hc_ = H[sl].clone().requires_grad_(True)
        pred = O.transform(batch["I_aug"][sl], Hc_, batch["patch_indices"][sl], 128)
        if loss_name == "l1_loss":
            part = (pred - batch["I2_aug"][sl]).abs().sum() / n_total
        else:
            part = O.ssim_map(pred, batch["I2_aug"][sl]).sum() / (B * 126 * 126)
        part.backward()
        g[sl] = Hc_.grad
    lt = udh.lib.LOSS_L1 if loss_name == "l1_loss" else udh.lib.LOSS_CUSTOM
    b = dev({k: (v.float() if isinstance(v, torch.Tensor) and v.dtype == torch.float64 else v) for k, v in batch.items()})
    Hc = H.float().cuda().contiguous()
    predc, sums = udh.ops.warp_loss_forward(b["I_aug"], Hc, b["I2_aug"], b["patch_indices"], 128, 128, want_pred=True)
    dpm = udh.ops.ssim_backward(predc, b["I2_aug"], 128, 128) if loss_name == "ssim_loss" else None
    dH = udh.ops.warp_loss_backward(b["I_aug"], Hc, b["I2_aug"], b["patch_indices"], 128, 128, lt, sums, dpred=dpm).cpu().double()
    g[:, 2, 2] = 0; dH[:, 2, 2] = 0                                         # h33 is a constant downstream
    errs = [rel_l2(dH[i], g[i]) for i in range(B)]
    worst = int(np.argmax(errs))
    print("warp backward %s B=128: worst per-sample rel L2 %.2e (sample %d), median %.2e" % (loss_name, errs[worst], worst, np.median(errs)))
    # d|pred - I2| flips sign wherever fp32 and fp64 disagree on the side of zero, so the l1 gradient is flip-limited: the
    # B = 3 bound of 5e-3 per sample is exceeded by the worst of 128 samples (measured 5.9e-3); the median pins the bulk
    assert errs[worst] < 1e-2 and np.median(errs) < 3e-3, (worst, dH[worst], g[worst])


@pytest.mark.parametrize("loss_type", ["h_loss", "l1_loss", "ssim_loss", "ncc_loss", "rec_loss", "l1_smooth_loss"])
def test_one_call_step_equals_separate_calls_B128(udh, loss_type):
    """test_gpu_parity.py's one-call step check at B = 128."""
    B = 128
    batch = dev(_batch(2, B))
    e1 = udh.engine.HomographyEngine(B, seed=1, loss_type=loss_type, lr=5e-4)
    e2 = udh.engine.HomographyEngine(B, seed=1, loss_type=loss_type, lr=5e-4)
    o1 = e1.forward(batch, train=True); e1.backward(batch, o1); g1 = e1.grads.clone(); d1 = e1.losses_dict(o1); e1.update()
    o2 = e2.train_step(batch); d2 = e2.losses_dict(o2)
    assert (o1["pred_h4p"] - o2["pred_h4p"]).abs().max().item() < 1e-6
    for k in d1:
        assert abs(d1[k] - d2[k]) <= 1e-5 * max(1.0, abs(d1[k])), k
    big = g1.abs() > 1e-3 * g1.abs().max()
    assert (e1.params - e2.params)[big].abs().max().item() <= 0.02 * 5e-4 and e2.global_step == 1
    assert rel_l2(e2.adam_m, e1.adam_m) < 1e-4
