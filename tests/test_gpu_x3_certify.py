"""The two-limb tensor-core kernels (UDH_NUMERIC_BF16X3, the mode bench.py and both CLIs run) on exact operands, against
float64 element by element, at the batch sizes the step runs (B in {1, 70, 128}: 70 leaves every two-tile item of the step's
two-tile instances half empty).  oracle/x3_limbs.py restates the number format:
  * integer operands: every product and partial sum is an exact integer, so forward (ReLU on and off, mask_out), dgrad
    (mask_bits), dW and db equal the stored-format value of float64 bit for bit: a lost, doubled or misplaced tile, item,
    slab, halo row or k-block shows with zero tolerance; the same through the single-pass bf16 kernels (their indexing);
  * limb operands (integer hi, lo = k 2^-10) with the lo limb on x only, on w / g only, or on both: each MMA pass checked
    alone and together, bit-exact against sum(hh + hl + lh) (the lo.lo term is excluded analytically), conv1_1's bias lo
    limb included;
  * the weight gradients at every grid shape (udh_set_sm_reserve(n), n in {0, 1, 7, 64, 127}) equal float64 exactly;
  * randn and wide-range operands (2^U(-24, 0), mixed signs): every element within its X.bound of float64;
  * the pool kernels of both tensor-core modes (udh_debug_tc_pool) bit-identical to oracle.simt_fp32's routing rule on tie
    windows, conv1_2's fused pool1 on flat integer inputs, and the two pool1 decision rules where they differ (fused: the
    fp32 accumulator; unfused: the stored hi + lo);
  * the engine at B = 128 on images with flat regions, layer by layer on its own inputs.
Each test prints its measured error or exact-match count next to what it asserts."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import oracle as O                                               # noqa: E402
from oracle import simt_fp32 as S                                            # noqa: E402
from oracle import x3_limbs as X                                             # noqa: E402
from _pool_ties import tie_windows                                           # noqa: E402


@pytest.fixture(scope="module")
def udh():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from unsuperviseddeephomographyral2018_b200 import _lib, engine, params
    _lib.require_device()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False

    class NS:
        pass
    ns = NS()
    ns.lib, ns.engine, ns.params, ns.L = _lib, engine, params, _lib.lib
    ns.sms = torch.cuda.get_device_properties(0).multi_processor_count
    return ns


P_ = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None

# the conv instances of the step (test_gpu_full_batch.LAYERS): (name, spatial size, cin, cout)
LAYERS = [("conv1_2", 128, 64, 64), ("conv2_x", 64, 64, 64), ("conv3_1", 32, 64, 128), ("conv3_2", 32, 128, 128),
          ("conv4_x", 16, 128, 128)]
BATCHES = [1, 70, 128]
LIMB_BATCHES = [1, 70]
RESERVES = [0, 1, 7, 64, 127]
POOLS = [("pool1", 128, 64), ("pool2", 64, 64), ("pool3", 32, 128)]         # (name, pre-pool size, channels)


def _T(cin, cout, dgrad):
    return 2 if (cin if dgrad else cout) == 64 else 1          # tiles per item of tc_conv_x3's instance


# ------------------------------------------------------------------------------------------------ kernels through the C ABI
def x3_conv(udh, x, w, bias, relu, dgrad, mask_bits=None, mask_out=None):
    B, H, W = x.shape[:3]
    cin, cout = w.shape[2], w.shape[3]
    out = torch.full((B, H, W, cin if dgrad else cout), float("nan"), device="cuda")
    scratch = torch.empty(udh.L.udh_debug_x3_scratch_bytes(B, H, W, cin, cout), device="cuda", dtype=torch.uint8)
    rc = udh.L.udh_debug_x3_conv_ex(P_(x), P_(w), P_(bias), P_(mask_bits), P_(mask_out), P_(out), P_(scratch), B, H, W, cin, cout,
                                    relu, dgrad, None)
    assert rc == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    return out


def x3_wgrad(udh, x, g):
    B, H, W, cin = x.shape
    cout = g.shape[3]
    dW = torch.zeros(3, 3, cin, cout, device="cuda"); db = torch.zeros(cout, device="cuda")
    scratch = torch.empty(udh.L.udh_debug_x3_scratch_bytes(B, H, W, cin, cout), device="cuda", dtype=torch.uint8)
    assert udh.L.udh_debug_x3_wgrad(P_(x), P_(g), P_(dW), P_(db), P_(scratch), B, H, W, cin, cout, None) == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    return dW, db


def x3_conv1(udh, x, w=None, bias=None, g=None, mask_out=None):
    """conv1_1 on x [B,H,W,2] (the two planes): forward (w, bias; mask words into mask_out) and / or weight gradient (g)."""
    B, H, W = x.shape[:3]
    I1, I2 = x[..., 0].contiguous(), x[..., 1].contiguous()
    out = torch.full((B, H, W, 64), float("nan"), device="cuda") if w is not None else None
    dW = torch.zeros(3, 3, 2, 64, device="cuda"); db = torch.zeros(64, device="cuda")
    scratch = torch.empty(udh.L.udh_debug_x3_scratch_bytes(B, H, W, 64, 64), device="cuda", dtype=torch.uint8)
    rc = udh.L.udh_debug_x3_conv1_ex(P_(I1), P_(I2), P_(w), P_(bias), P_(mask_out), P_(out), P_(g), P_(dW) if g is not None else None,
                                     P_(db) if g is not None else None, P_(scratch), B, H, W, None)
    assert rc == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    return out, dW, db


def x3_rows(udh, x, w, bias, rows, mask_bits=None):
    B, H, W = x.shape[:3]
    if rows == 1:
        out = torch.full((B, H // 2, W // 2, 64), float("nan"), device="cuda")
        codes = torch.full((B, H // 2, W // 2, 8), -1, device="cuda", dtype=torch.int32)
    else:
        out, codes = torch.full((B, H, W, 64), float("nan"), device="cuda"), None
    scratch = torch.empty(udh.L.udh_debug_x3_scratch_bytes(B, H, W, 64, 64), device="cuda", dtype=torch.uint8)
    rc = udh.L.udh_debug_x3_conv_rows(P_(x), P_(w), P_(bias), P_(mask_bits), P_(out), P_(codes), P_(scratch), B, H, W, rows, None)
    assert rc == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    return out, codes


def tc_pool(udh, mode, x, dout):
    """udh_debug_tc_pool: forward of x, then backward of dout from the forward's codes."""
    B, H, W, C = x.shape
    out = torch.full((B, H // 2, W // 2, C), float("nan"), device="cuda")
    codes = torch.full((B, H // 2, W // 2, C // 8), -1, device="cuda", dtype=torch.int32)
    din = torch.full_like(x, float("nan"))
    rc = udh.L.udh_debug_tc_pool(mode, P_(x), P_(out), P_(codes), P_(dout), P_(din), B, H, W, C, None)
    assert rc == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    return out, codes, din


# ------------------------------------------------------------------------------------------------ float64 references
def ref_conv(x, w, bias=None, dgrad=False):
    wk = torch.flip(w, dims=(0, 1)).permute(2, 3, 0, 1) if dgrad else w.permute(3, 2, 0, 1)
    r = F.conv2d(x.double().permute(0, 3, 1, 2), wk.double().contiguous(), None if bias is None else bias.double(), padding=1)
    return r.permute(0, 2, 3, 1)


def ref_wgrad(x, g):
    dW = torch.nn.grad.conv2d_weight(x.double().permute(0, 3, 1, 2), (g.shape[3], x.shape[3], 3, 3), g.double().permute(0, 3, 1, 2),
                                     padding=1)
    return dW.permute(2, 3, 1, 0), g.double().sum(dim=(0, 1, 2))


def _where(shape, flat_idx):
    return tuple(int(v) for v in np.unravel_index(int(flat_idx), tuple(shape)))


def check_exact(got, want, what, T=None, rows=False, names="n,y,x,c"):
    """got == want element by element (values; the sign of a zero is not compared).  A failure names the image and position
    and, for conv outputs, the 128-row tile and the item of the padded stream (rows: the row-tile item)."""
    got, want = got.double(), want.double()
    bad = got != want
    if bad.any():
        idx = bad.flatten().nonzero().flatten()[:4].tolist()
        msgs = []
        for i in idx:
            pos = _where(want.shape, i)
            m = "(%s)=%s: %r vs %r" % (names, pos, got.flatten()[i].item(), want.flatten()[i].item())
            if T is not None:
                n, y, x = pos[:3]
                Hh, Ww = want.shape[1], want.shape[2]
                q = (n * (Hh + 2) + y + 1) * (Ww + 2) + x + 1
                m += ", tile %d, item %d" % (q // 128, q // 128 // T)
            elif rows:
                m += ", item %d" % (pos[0] * (want.shape[1] // 2) + pos[1] // 2)
            msgs.append(m)
        nimg = len(set(_where(want.shape, i)[0] for i in bad.flatten().nonzero().flatten()[:100000].tolist()))
        pytest.fail("%s: %d elements (in >= %d images or rows) differ: %s" % (what, int(bad.sum()), nimg, "; ".join(msgs)))
    return int(got.numel())


def check_bound(got, ref, bound, what, names="n,y,x,c"):
    d = (got.double() - ref).abs()
    bad = d > bound
    if bad.any():
        frac = torch.where(bad, d / bound.clamp_min(1e-300), torch.zeros_like(d)).flatten()
        idx = frac.topk(min(4, int(bad.sum()))).indices.tolist()
        pytest.fail("%s: %d elements over the bound: %s" % (what, int(bad.sum()), "; ".join(
            "(%s)=%s: err %.3e > bound %.3e" % (names, _where(ref.shape, i), d.flatten()[i].item(), bound.flatten()[i].item())
            for i in idx)))
    pos = bound > 0
    return (d[pos] / bound[pos]).max().item() if pos.any() else 0.0


def decode_codes(codes, C):
    sh = (torch.arange(C, device="cuda") % 8) * 3
    return (codes.long()[..., torch.arange(C, device="cuda") // 8] >> sh) & 7              # [B,H/2,W/2,C]


def rule_codes(v):
    """The routing rule's code of every window of v (oracle.simt_fp32.pool_bwd): index 0-3 of the first maximum in row-major
    order, 4 where the maximum is not > 0."""
    din = S.pool_bwd(v, torch.ones(S.pool_fwd(v).shape, dtype=v.dtype, device=v.device))
    win = torch.stack(S._windows(din), dim=-1)                                             # [B,H/2,W/2,C,4]
    return torch.where(win.sum(dim=-1) > 0, win.argmax(dim=-1), torch.full(win.shape[:-1], 4, device=v.device))


def tie_counts(v):
    a, b, c, d = S._windows(v)
    m = S.pool_fwd(v)
    ties = ((a == m).int() + (b == m).int() + (c == m).int() + (d == m).int() >= 2) & (m > 0)
    return int(ties.sum()), int((m <= 0).sum())


def mask_words(gen, B, H, W, C):
    """Random uint32 mask words over the padded positions and the {0,1} mask they encode on the interior."""
    words = torch.randint(-2 ** 31, 2 ** 31, (B, H + 2, W + 2, C // 32), device="cuda", generator=gen, dtype=torch.int64)
    bits = (words[..., None] >> torch.arange(32, device="cuda")) & 1
    m = bits.reshape(B, H + 2, W + 2, C)[:, 1:H + 1, 1:W + 1].double()
    return words.to(torch.int32).contiguous(), m


def mask_of(out):
    B, H, W, C = out.shape
    bits = (out > 0).long().reshape(B, H, W, C // 32, 32) << torch.arange(32, device="cuda")
    words = torch.zeros(B, H + 2, W + 2, C // 32, device="cuda", dtype=torch.int64)
    words[:, 1:H + 1, 1:W + 1] = bits.sum(dim=-1)
    return words.to(torch.int32)


# ------------------------------------------------------------------------------------------------ 1. integer operands, two limbs
@pytest.mark.parametrize("mode", ["fwd_relu", "fwd_linear", "dgrad"])
@pytest.mark.parametrize("name,H,cin,cout", LAYERS)
@pytest.mark.parametrize("B", BATCHES)
def test_x3_conv_integer_operands_bit_exact(udh, B, name, H, cin, cout, mode):
    dgrad, relu = int(mode == "dgrad"), int(mode == "fwd_relu")
    gen = torch.Generator(device="cuda").manual_seed(B * 1000 + H + cin + 7 * dgrad + relu)
    x = X.int_operand(gen, (B, H, H, cout if dgrad else cin)); w = X.int_operand(gen, (3, 3, cin, cout))
    bias = None if dgrad else X.int_operand(gen, (cout,), 3)
    ref = ref_conv(x, w, bias, dgrad)
    X.require_exact(ref_conv(x.abs(), w.abs(), None if bias is None else bias.abs(), dgrad), 1.0, name)
    what = "x3 %s %s B=%d (integer operands)" % (name, mode, B)
    T = _T(cin, cout, dgrad)
    if dgrad:
        words, m = mask_words(gen, B, H, H, cin)
        out = x3_conv(udh, x, w, None, 0, 1, mask_bits=words)
        n = check_exact(out, X.stored(ref) * m, what + " + mask_bits", T)
    else:
        mo = torch.full((B * (H + 2) * (H + 2), cout // 32), -1, device="cuda", dtype=torch.int32)
        out = x3_conv(udh, x, w, bias, relu, 0, mask_out=mo)
        n = check_exact(out, X.stored(F.relu(ref) if relu else ref), what, T)
        assert torch.equal(mo, mask_of(out).reshape(mo.shape)), "%s: mask_out differs from out > 0" % what
    print("%s: %d elements bit-exact (T=%d)%s" % (what, n, T, ", mask_out == out > 0" if not dgrad else ""))


@pytest.mark.parametrize("name,H,cin,cout", LAYERS)
@pytest.mark.parametrize("B", BATCHES)
def test_x3_wgrad_integer_operands_bit_exact(udh, B, name, H, cin, cout):
    gen = torch.Generator(device="cuda").manual_seed(B * 77 + H + cin)
    x = X.int_operand(gen, (B, H, H, cin), 1); g = X.int_operand(gen, (B, H, H, cout), 1)
    rW, rb = ref_wgrad(x, g)
    X.require_exact(ref_wgrad(x.abs(), g.abs())[0], 1.0, name + " dW"); X.require_exact(g.abs().double().sum(dim=(0, 1, 2)), 1.0, name + " db")
    dW, db = x3_wgrad(udh, x, g)
    what = "x3 %s wgrad B=%d (integer operands)" % (name, B)
    n = check_exact(dW, rW, what + " dW", names="ky,kx,ci,co") + check_exact(db, rb, what + " db", names="co")
    print("%s: dW and db bit-exact (%d elements, max |dW| %d)" % (what, n, int(rW.abs().max())))


@pytest.mark.parametrize("B", BATCHES)
def test_x3_conv1_1_integer_operands_bit_exact(udh, B):
    H = 128
    gen = torch.Generator(device="cuda").manual_seed(B * 5 + 3)
    x = X.int_operand(gen, (B, H, H, 2)); w = X.int_operand(gen, (3, 3, 2, 64)); bias = X.int_operand(gen, (64,), 3)
    mo = torch.full((B, H + 2, H + 2, 2), -1, device="cuda", dtype=torch.int32)
    out, _, _ = x3_conv1(udh, x, w, bias, mask_out=mo)
    n = check_exact(out, X.stored(F.relu(ref_conv(x, w, bias))), "x3 conv1_1 fwd B=%d (integer operands)" % B)
    inner = (slice(None), slice(1, H + 1), slice(1, H + 1))           # the kernel writes the words of interior positions
    assert torch.equal(mo[inner], mask_of(out)[inner]), "x3 conv1_1 B=%d: %d mask_out words differ from out > 0" % (
        B, int((mo[inner] != mask_of(out)[inner]).sum()))
    x = X.int_operand(gen, (B, H, H, 2), 1); g = X.int_operand(gen, (B, H, H, 64), 1)
    rW, rb = ref_wgrad(x, g)
    _, dW, db = x3_conv1(udh, x, g=g)
    check_exact(dW, rW, "x3 conv1_1 dW B=%d" % B, names="ky,kx,ci,co"); check_exact(db, rb, "x3 conv1_1 db B=%d" % B, names="co")
    print("x3 conv1_1 B=%3d (integer operands): forward (%d elements), mask_out == out > 0, dW and db bit-exact" % (B, n))


def _flat_int(gen, B, H, W, C, lo=0, hi=2, block=8):
    """Integer input constant on block x block squares: the conv outputs of a square's interior are equal, so pool windows
    there tie."""
    x = torch.randint(lo, hi + 1, (B, H // block, W // block, C), device="cuda", generator=gen).float()
    return x.repeat_interleave(block, dim=1).repeat_interleave(block, dim=2).contiguous()


@pytest.mark.parametrize("B", BATCHES)
def test_x3_rows_fused_pool1_and_dgrad_integer_bit_exact(udh, B):
    """conv1_2's row-tile kernels: the fused conv + pool1 on flat integer inputs (ties are common) gives the stored maximum
    and the code of the first maximum of the exact post-ReLU accumulators; the row-tile dgrad with conv1_1's mask fused is
    bit-exact."""
    H = 128
    gen = torch.Generator(device="cuda").manual_seed(B * 13 + 1)
    x = _flat_int(gen, B, H, H, 64); w = X.int_operand(gen, (3, 3, 64, 64), 1); bias = X.int_operand(gen, (64,), 3)
    post = F.relu(ref_conv(x, w, bias))
    pooled, codes = x3_rows(udh, x, w, bias, 1)
    check_exact(pooled, X.stored(S.pool_fwd(post)), "x3 conv1_2 + pool1 rows B=%d: pooled" % B, rows=True)
    k, want = decode_codes(codes, 64), rule_codes(post)
    bad = k != want
    assert not bad.any(), "x3 conv1_2 + pool1 rows B=%d: %d codes differ from the rule, first at (n,y,x,c)=%s" % (
        B, int(bad.sum()), _where(want.shape, bad.flatten().nonzero()[0].item()))
    ties, zeros = tie_counts(post)
    windows = want.numel()
    assert ties > windows // 20, (ties, windows)
    g = X.int_operand(gen, (B, H, H, 64)); w2 = X.int_operand(gen, (3, 3, 64, 64))
    words, m = mask_words(gen, B, H, H, 64)
    out, _ = x3_rows(udh, g, w2, None, 2, mask_bits=words)
    check_exact(out, X.stored(ref_conv(g, w2, None, True)) * m, "x3 conv1_2 dgrad rows + mask B=%d" % B, rows=True)
    print("x3 conv1_2 rows B=%3d: pooled and %d codes exact (%d tied positive maxima, %d non-positive windows); dgrad + mask exact"
          % (B, windows, ties, zeros))


# ------------------------------------------------------------------------------------------------ 2. integer operands, bf16 mode
@pytest.mark.parametrize("mode", ["fwd_relu", "dgrad", "wgrad"])
@pytest.mark.parametrize("name,H,cin,cout", LAYERS)
@pytest.mark.parametrize("B", BATCHES)
def test_bf16_integer_operands_bit_exact(udh, B, name, H, cin, cout, mode):
    """The single-pass bf16 kernels' indexing: integer operands are bf16 values, so the fp32 outputs equal float64 exactly."""
    gen = torch.Generator(device="cuda").manual_seed(B * 999 + H + cin)
    scratch = torch.empty(udh.L.udh_debug_tc_conv_scratch_bytes(B, H, H, cin, cout), device="cuda", dtype=torch.uint8)
    what = "bf16 %s %s B=%d (integer operands)" % (name, mode, B)
    if mode == "wgrad":
        x = X.int_operand(gen, (B, H, H, cin), 1); g = X.int_operand(gen, (B, H, H, cout), 1)
        dW = torch.zeros(3, 3, cin, cout, device="cuda"); db = torch.zeros(cout, device="cuda")
        assert udh.L.udh_debug_tc_wgrad(P_(x), P_(g), P_(dW), P_(db), P_(scratch), B, H, H, cin, cout, None) == 0, udh.L.udh_last_error()
        torch.cuda.synchronize()
        rW, rb = ref_wgrad(x, g)
        check_exact(dW, rW, what + " dW", names="ky,kx,ci,co"); check_exact(db, rb, what + " db", names="co")
    else:
        dgrad = int(mode == "dgrad")
        x = X.int_operand(gen, (B, H, H, cout if dgrad else cin)); w = X.int_operand(gen, (3, 3, cin, cout))
        bias = None if dgrad else X.int_operand(gen, (cout,), 3)
        out = torch.full((B, H, H, cin if dgrad else cout), float("nan"), device="cuda")
        rc = udh.L.udh_debug_tc_conv(P_(x), P_(w), P_(bias), P_(out), P_(scratch), B, H, H, cin, cout, 1 - dgrad, dgrad, None)
        assert rc == 0, udh.L.udh_last_error()
        torch.cuda.synchronize()
        ref = ref_conv(x, w, bias, dgrad)
        check_exact(out, ref if dgrad else F.relu(ref), what, _T(cin, cout, dgrad))
    print("%s: bit-exact" % what)


@pytest.mark.parametrize("B", BATCHES)
def test_bf16_conv_pool_integer_bit_exact(udh, B):
    H = 128
    gen = torch.Generator(device="cuda").manual_seed(B * 31 + 5)
    x = _flat_int(gen, B, H, H, 64); w = X.int_operand(gen, (3, 3, 64, 64), 1); bias = X.int_operand(gen, (64,), 3)
    pooled = torch.full((B, H // 2, H // 2, 64), float("nan"), device="cuda")
    codes = torch.full((B, H // 2, H // 2, 8), -1, device="cuda", dtype=torch.int32)
    scratch = torch.empty(udh.L.udh_debug_tc_conv_scratch_bytes(B, H, H, 64, 64), device="cuda", dtype=torch.uint8)
    assert udh.L.udh_debug_tc_conv_pool(P_(x), P_(w), P_(bias), P_(pooled), P_(codes), P_(scratch), B, H, H, None) == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    post = F.relu(ref_conv(x, w, bias))
    check_exact(pooled, X.stored(S.pool_fwd(post), "bf16"), "bf16 conv1_2 + pool1 B=%d: pooled" % B, rows=True)
    assert torch.equal(decode_codes(codes, 64), rule_codes(post)), "bf16 conv1_2 + pool1 B=%d: codes differ from the rule" % B
    print("bf16 conv1_2 + pool1 B=%3d: pooled and codes exact (%d tied positive maxima)" % (B, tie_counts(post)[0]))


# ------------------------------------------------------------------------------------------------ 3. limb operands
LIMB = {"x": (True, False), "w": (False, True), "both": (True, True)}       # which operand carries a lo limb


@pytest.mark.parametrize("limb", list(LIMB))
@pytest.mark.parametrize("name,H,cin,cout", LAYERS)
@pytest.mark.parametrize("B", LIMB_BATCHES)
def test_x3_conv_limb_operands_bit_exact(udh, B, name, H, cin, cout, limb):
    """Forward (linear) and dgrad with the lo limb on the activation only (the lo.hi pass), on the weight only (hi.lo), or on
    both: bit-exact against the stored value of sum(hh + hl + lh) + bias."""
    lx, lw = LIMB[limb]
    gen = torch.Generator(device="cuda").manual_seed(B * 7 + H + cin + len(limb))
    res = []
    for dgrad in (0, 1):
        x = X.limb_operand(gen, (B, H, H, cout if dgrad else cin), lx, vmax=2)
        w = X.limb_operand(gen, (3, 3, cin, cout), lw, vmax=1)
        bias = None if dgrad else X.int_operand(gen, (cout,), 2)
        terms = X.abs_terms(lambda a, b: ref_conv(a, b, None, dgrad), x, w) + (0 if bias is None else bias.double().abs())
        grid = X.require_exact(terms, X.GRID_LO, name)
        want = X.three_pass(lambda a, b: ref_conv(a, b, None, dgrad), x, w) + (0 if bias is None else bias.double())
        out = x3_conv(udh, x, w, bias, 0, dgrad)
        check_exact(out, X.stored(want), "x3 %s %s B=%d (lo on %s)" % (name, "dgrad" if dgrad else "fwd", B, limb), _T(cin, cout, dgrad))
        res.append(grid)
    print("x3 %-8s B=%3d lo on %-4s: forward and dgrad bit-exact (sum |terms| <= %.2e grid units)" % (name, B, limb, max(res)))


WGRAD_INSTANCES = [("conv1_1", 128, 2, 64)] + LAYERS


def _wgrad_any(udh, name, x, g):
    return x3_conv1(udh, x, g=g)[1:] if name == "conv1_1" else x3_wgrad(udh, x, g)


@pytest.mark.parametrize("limb", ["x", "g", "both"])
@pytest.mark.parametrize("name,H,cin,cout", WGRAD_INSTANCES)
@pytest.mark.parametrize("B", LIMB_BATCHES)
def test_x3_wgrad_limb_operands_bit_exact(udh, B, name, H, cin, cout, limb):
    """dW bit-exact against sum(hh + hl + lh) and db against sum g (ones . (g_hi + g_lo)).  g is sparse so that every
    partial sum stays below 2^22 grid units.  conv1_1's weight gradient adds the lo.lo term as well, so it is checked with
    the lo limb on one side only."""
    if name == "conv1_1" and limb == "both":
        pytest.skip("conv1_1's weight gradient adds x_lo.g_lo too: with both lo limbs the sum leaves the 2^-10 grid")
    lx, lg = limb in ("x", "both"), limb in ("g", "both")
    gen = torch.Generator(device="cuda").manual_seed(B * 11 + H + cin + len(limb))
    x = X.limb_operand(gen, (B, H, H, cin), lx, vmax=1)
    g = X.limb_operand(gen, (B, H, H, cout), lg, vmax=1, density=min(1.0, 1024.0 / (1.5 * B * H * H)))
    grid = max(X.require_exact(X.abs_terms(lambda a, b: ref_wgrad(a, b)[0], x, g), X.GRID_LO, name + " dW"),
               X.require_exact(g.abs().double().sum(dim=(0, 1, 2)), X.GRID_LO, name + " db"))
    rW = X.three_pass(lambda a, b: ref_wgrad(a, b)[0], x, g)
    rb = g.double().sum(dim=(0, 1, 2))
    dW, db = _wgrad_any(udh, name, x, g)
    what = "x3 %s wgrad B=%d (lo on %s)" % (name, B, limb)
    check_exact(dW, rW, what + " dW", names="ky,kx,ci,co"); check_exact(db, rb, what + " db", names="co")
    print("%s: dW and db bit-exact (sum |terms| <= %.2e grid units, %d non-zero g)" % (what, grid, int((g != 0).sum())))


@pytest.mark.parametrize("limb", ["x", "w", "both", "bias"])
@pytest.mark.parametrize("B", LIMB_BATCHES)
def test_x3_conv1_1_limb_operands_bit_exact(udh, B, limb):
    """conv1_1's forward with the lo limb on the images, the weights, both, or the bias (its bias-lo weight column)."""
    H = 128
    gen = torch.Generator(device="cuda").manual_seed(B * 3 + len(limb))
    x = X.limb_operand(gen, (B, H, H, 2), limb in ("x", "both"))
    w = X.limb_operand(gen, (3, 3, 2, 64), limb in ("w", "both"))
    bias = X.limb_operand(gen, (64,), limb == "bias", vmax=3)
    bias_terms = X.split(bias)[0].double().abs() + X.split(bias)[1].double().abs()           # hi.b_hi + hi.b_lo of the ones column
    X.require_exact(X.abs_terms(lambda a, b: ref_conv(a, b), x, w) + bias_terms, X.GRID_LO, "conv1_1")
    want = F.relu(X.three_pass(lambda a, b: ref_conv(a, b), x, w) + bias.double())
    out, _, _ = x3_conv1(udh, x, w, bias)
    n = check_exact(out, X.stored(want), "x3 conv1_1 fwd B=%d (lo on %s)" % (B, limb))
    print("x3 conv1_1 B=%3d lo on %-4s: %d elements bit-exact" % (B, limb, n))


# ------------------------------------------------------------------------------------------------ 4. every grid shape
@pytest.fixture
def sm_reserve(udh):
    def set_(n):
        assert udh.L.udh_set_sm_reserve(n) == 0, udh.L.udh_last_error()
    yield set_
    udh.L.udh_set_sm_reserve(0)


@pytest.mark.parametrize("name,H,cin,cout", WGRAD_INSTANCES)
def test_x3_wgrad_exact_at_every_grid_shape(udh, sm_reserve, name, H, cin, cout):
    """With integer operands dW and db do not depend on the order of summation: they equal float64 at every SM reserve, so
    every item and slab of every partition is summed exactly once."""
    B = 128
    gen = torch.Generator(device="cuda").manual_seed(H * 3 + cin)
    x = X.int_operand(gen, (B, H, H, cin), 1); g = X.int_operand(gen, (B, H, H, cout), 1)
    rW, rb = ref_wgrad(x, g)
    for n in RESERVES:
        sm_reserve(n)
        dW, db = _wgrad_any(udh, name, x, g)
        check_exact(dW, rW, "x3 %s dW, %d SMs reserved" % (name, n), names="ky,kx,ci,co")
        check_exact(db, rb, "x3 %s db, %d SMs reserved" % (name, n), names="co")
    print("x3 %-8s wgrad B=128: dW and db bit-exact at SM reserve %s" % (name, RESERVES))


# ------------------------------------------------------------------------------------------------ 5. per-element bound
def _real(gen, shape, kind, scale=1.0):
    if kind == "randn":
        return (torch.randn(shape, device="cuda", generator=gen) * scale).contiguous()
    mag = torch.pow(2.0, -24.0 * torch.rand(shape, device="cuda", generator=gen))       # 2^U(-24, 0), mixed signs
    return (mag * torch.where(torch.rand(shape, device="cuda", generator=gen) < 0.5, -1.0, 1.0) * scale).contiguous()


def wgrad_chain(sms, name, B, H, cin, cout):
    """(k-steps of the longest accumulator chain, slabs summed after it) of the launcher's partition on a grid of sms SMs."""
    if name == "conv1_1":
        tiles = B * H
        grid = min(tiles, 2 * sms)
        return -(-tiles // grid) * 8 * 2, grid + 1               # 8 k-steps per 128-pixel tile and G limb; x_hi + x_lo add
    T = 2 if cout == 64 else 1
    items = -(-(-(-(B * (H + 2) * (H + 2)) // 128)) // T)   # items of T 128-position tiles
    if cout == 64:
        per = min(items, sms // 2)                          # CTAs per group of the N = 192 kernel
    else:
        per = max(1, sms // (5 if cin == 64 else 10))       # at least this many CTAs per group of the generic kernel
    return -(-items // per) * (T * 128 // 16) * 3, per + 1


@pytest.mark.parametrize("kind", ["randn", "wide"])
@pytest.mark.parametrize("name,H,cin,cout", WGRAD_INSTANCES)
@pytest.mark.parametrize("B", BATCHES)
def test_x3_within_per_element_bound_of_fp64(udh, sm_reserve, B, name, H, cin, cout, kind):
    """Every element within X.bound of float64.  At B = 128 the weight gradients are also run with 127 SMs reserved, where
    a CTA's accumulator chain is longest."""
    gen = torch.Generator(device="cuda").manual_seed(B * 17 + H + cin + len(kind))
    fr = {}
    x = _real(gen, (B, H, H, cin), kind)
    w = _real(gen, (3, 3, cin, cout), kind, 1.0 / (3 * cin ** 0.5))
    bias = _real(gen, (cout,), kind, 0.1)
    g = _real(gen, (B, H, H, cout), kind, 0.1)
    if name == "conv1_1":
        out = x3_conv1(udh, x, w, bias)[0]
        ref = F.relu(ref_conv(x, w, bias))
        fr["fwd"] = check_bound(out, ref, X.bound(ref_conv(x.abs(), w.abs(), bias.abs()), X.chain_gamma(6, 0), ref), "x3 conv1_1 fwd")
    else:
        out = x3_conv(udh, x, w, bias, 0, 0)
        ref = ref_conv(x, w, bias)
        fr["fwd"] = check_bound(out, ref, X.bound(ref_conv(x.abs(), w.abs(), bias.abs()), X.chain_gamma(27 * cin // 16, 1), ref),
                                "x3 %s fwd B=%d %s" % (name, B, kind))
        out = x3_conv(udh, g, w, None, 0, 1)
        ref = ref_conv(g, w, None, True)
        fr["dgrad"] = check_bound(out, ref, X.bound(ref_conv(g.abs(), w.abs(), None, True), X.chain_gamma(27 * cout // 16), ref),
                                  "x3 %s dgrad B=%d %s" % (name, B, kind))
    rW, rb = ref_wgrad(x, g)
    aW, ab = ref_wgrad(x.abs(), g.abs())[0], g.abs().double().sum(dim=(0, 1, 2))
    chains = []
    for n in ([0, 127] if B == 128 else [0]):
        sm_reserve(n)
        L, m = wgrad_chain(max(udh.sms - n, 1), name, B, H, cin, cout)
        gm = X.chain_gamma(L, m)
        dW, db = _wgrad_any(udh, name, x, g)
        tag = "" if n == 0 else " reserve %d" % n
        fr["dW" + tag] = check_bound(dW, rW, X.bound(aW, gm), "x3 %s dW B=%d %s%s" % (name, B, kind, tag), "ky,kx,ci,co")
        fr["db" + tag] = check_bound(db, rb, X.bound(ab, gm), "x3 %s db B=%d %s%s" % (name, B, kind, tag), "co")
        chains.append("%d k-steps + %d slabs%s" % (L, m, tag))
    print("x3 %-8s B=%3d %-5s: worst fraction of the per-element bound %s (wgrad chain %s)"
          % (name, B, kind, ", ".join("%s %.3f" % kv for kv in fr.items()), "; ".join(chains)))
    assert max(fr.values()) <= 1.0


# ------------------------------------------------------------------------------------------------ 6. pools
@pytest.mark.parametrize("mode", ["bf16x3", "bf16"])
@pytest.mark.parametrize("name,H,C", POOLS)
@pytest.mark.parametrize("B", [1, 128])
def test_tc_pool_routing_rule_on_ties(udh, B, name, H, C, mode):
    """The step's pool kernels of each tensor-core mode on windows of 2, 3 and 4 equal maxima, all-zero and +-0 windows:
    pooled values, codes and the routed gradient bit-identical to the rule applied to the stored values."""
    nm = udh.lib.NUMERIC_BF16X3 if mode == "bf16x3" else udh.lib.NUMERIC_BF16
    gen = torch.Generator(device="cuda").manual_seed(B * 31 + H + C + len(mode))
    x = tie_windows(gen, B, H, H, C)
    dout = torch.randn(B, H // 2, H // 2, C, device="cuda", generator=gen)
    dout[..., 0] = -0.0
    out, codes, din = tc_pool(udh, nm, x, dout)
    xs, ds = X.stored(x, mode), X.stored(dout, mode)
    check_exact(out, S.pool_fwd(xs), "%s %s B=%d forward" % (mode, name, B))
    k, want = decode_codes(codes, C), rule_codes(xs)
    assert torch.equal(k, want), "%s %s B=%d: %d codes differ from the rule" % (mode, name, B, int((k != want).sum()))
    rb = S.pool_bwd(xs, ds)
    bad = din.view(torch.int32) != rb.view(torch.int32)
    assert not bad.any(), "%s %s B=%d backward: %d elements differ from the rule, first at (n,y,x,c)=%s" % (
        mode, name, B, int(bad.sum()), _where(x.shape, bad.flatten().nonzero()[0].item()))
    ties, zeros = tie_counts(xs)
    windows = want.numel()
    assert ties > windows // 3 and zeros > windows // 10, (ties, zeros, windows)
    print("%s %s B=%3d: forward, codes and routing bit-identical to the rule on %d windows (%d tied positive maxima, %d zero)"
          % (mode, name, B, windows, ties, zeros))


@pytest.mark.parametrize("B", [1, 70])
def test_x3_pool1_fused_and_unfused_rules_where_they_differ(udh, B):
    """Accumulators 160 + j 2^-10 with 256 <= j < 512 are distinct in fp32 but an odd j splits to the same hi + lo as its even
    neighbour.  conv1_2's fused epilogue decides on the fp32 accumulator, the unfused path (generic conv, then pool_fwd_x3)
    on the stored hi + lo: each follows its own rule exactly, and every fused code points at a maximum of the stored values."""
    H = 128
    gen = torch.Generator(device="cuda").manual_seed(B + 4242)
    # x = 2 + k 2^-10 everywhere (k in -3..3, below half an ulp of 2), w integer in {-1, 0, 1}: the integer part of every
    # interior accumulator is 2 sum(w) of its channel, the rest sum(k w) 2^-10; the bias moves it to 160 + (300 + j) 2^-10
    k = torch.randint(-3, 4, (B, H, H, 64), device="cuda", generator=gen).float()
    x = (2.0 + k * X.GRID_LO).contiguous()
    assert torch.equal(X.split(x)[0], torch.full_like(x, 2.0)) and torch.equal(X.split(x)[1], k * X.GRID_LO)
    w = X.int_operand(gen, (3, 3, 64, 64), 1)
    bias = (160.0 - 2.0 * w.sum(dim=(0, 1, 2)) + 300 * X.GRID_LO).contiguous()
    X.require_exact(X.abs_terms(lambda a, b: ref_conv(a, b), x, w) + bias.double().abs(), X.GRID_LO, "conv1_2")
    post = F.relu(ref_conv(x, w, bias))                                  # exact: the fp32 accumulators the fused path sees
    st = X.stored(post)
    pooled, codes_f = x3_rows(udh, x, w, bias, 1)
    full = x3_conv(udh, x, w, bias, 1, 0)
    check_exact(full, st, "x3 conv1_2 generic B=%d" % B)
    _, codes_u, _ = tc_pool(udh, udh.lib.NUMERIC_BF16X3, full, torch.zeros(B, H // 2, H // 2, 64, device="cuda"))
    kf, ku = decode_codes(codes_f, 64), decode_codes(codes_u, 64)
    rf, ru = rule_codes(post), rule_codes(st)
    assert torch.equal(kf, rf), "fused pool1: %d codes differ from the fp32-accumulator rule" % int((kf != rf).sum())
    assert torch.equal(ku, ru), "unfused pool1: %d codes differ from the stored-value rule" % int((ku != ru).sum())
    check_exact(pooled, S.pool_fwd(st), "x3 conv1_2 + pool1 rows B=%d: pooled" % B, rows=True)
    win = torch.stack(S._windows(st), dim=-1)
    picked = torch.gather(win, 4, kf.clamp(max=3).unsqueeze(-1)).squeeze(-1)
    live = kf < 4
    assert torch.equal(picked[live], S.pool_fwd(st)[live]), "a fused code points at a non-maximum of the stored values"
    differ = int((kf != ku).sum())
    assert differ > 0, "no window where the two rules differ: the construction does not reach the case"
    print("pool1 B=%3d: fused codes follow the fp32 rule, unfused the stored rule, exactly; they differ in %d of %d windows, "
          "every fused code at a stored maximum" % (B, differ, kf.numel()))


# ------------------------------------------------------------------------------------------------ 7. the engine on its own gates
def _flat_batch(seed, B):
    batch = O.make_batch(seed, B)
    for k in ("I1_aug", "I2_aug"):
        t = batch[k].clone()
        t[:, 16:64, 32:96] = 1.5
        t[:, 80:, :42] = -1.25
        batch[k] = t
    return batch


def test_x3_engine_B128_layer_by_layer_on_its_own_inputs(udh):
    """A bf16x3 engine at B = 128 on the unfused path, images with flat regions: each conv activation within its per-element
    bound of float64 applied to the engine's own materialised input; pool2 and pool3 equal the rule on the stored pre-pool
    activations; udh_debug_tc_pool on those activations reproduces the rule."""
    B = 128
    udh.L.udh_debug_x3_set_rows(0)
    try:
        eng = udh.engine.HomographyEngine(B, seed=None, numeric="bf16x3")
        eng.load_flat(udh.params.init_flat_large(2))
        batch = _flat_batch(2, B)
        db = {k: (v.cuda().contiguous() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}
        eng.forward(db, train=False)
        eng.materialize_activations()
        torch.cuda.synchronize()
        specs = [(2, 1, 64), (64, 1, 64), (64, 2, 64), (64, 2, 64), (64, 4, 128), (128, 4, 128), (128, 8, 128), (128, 8, 128)]
        acts = {i: eng.activation(i).reshape(B, 128 // d, 128 // d, c) for i, (_, d, c) in enumerate(specs)}
        acts.update({8: eng.activation(8).reshape(B, 64, 64, 64), 9: eng.activation(9).reshape(B, 32, 32, 64),
                     10: eng.activation(10).reshape(B, 16, 16, 128)})
        p = eng.named_parameters()
        names = list(p)
        I = torch.cat([db["I1_aug"], db["I2_aug"]], dim=3)
        report = []
        for i in range(8):
            x = I if i == 0 else (acts[8 + (i - 2) // 2] if i in (2, 4, 6) else acts[i - 1])
            w, b = p[names[2 * i]], p[names[2 * i + 1]]
            ref = F.relu(ref_conv(x, w, b))
            cin = specs[i][0]
            g_ = X.chain_gamma(6, 0) if i == 0 else X.chain_gamma(27 * cin // 16, 1)
            frac = check_bound(acts[i], ref, X.bound(ref_conv(x.abs(), w.abs(), b.abs()), g_, ref), "engine conv layer %d" % i)
            report.append("conv%d %.3f" % (i, frac))
        gen = torch.Generator(device="cuda").manual_seed(9)
        for pi, src in ((8, 1), (9, 3), (10, 5)):
            check_exact(acts[pi], S.pool_fwd(acts[src]), "engine pool%d" % (pi - 7))
            pre = acts[src].contiguous()
            dout = torch.randn(acts[pi].shape, device="cuda", generator=gen)
            out, codes, din = tc_pool(udh, udh.lib.NUMERIC_BF16X3, pre, dout)
            check_exact(out, S.pool_fwd(pre), "entry pool%d on the engine's activations" % (pi - 7))
            assert torch.equal(decode_codes(codes, pre.shape[3]), rule_codes(pre)), pi
            assert torch.equal(din.view(torch.int32), S.pool_bwd(pre, X.stored(dout)).view(torch.int32)), pi
            ties, zeros = tie_counts(pre)
            assert ties > 0, pi
            report.append("pool%d exact (%d tied positive maxima, %d non-positive windows)" % (pi - 7, ties, zeros))
        print("bf16x3 engine B=128 (unfused), fraction of the per-element bound: %s" % ", ".join(report))
        del eng
    finally:
        udh.L.udh_debug_x3_set_rows(1)
