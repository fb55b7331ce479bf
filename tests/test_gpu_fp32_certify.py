"""The fp32 CUDA-core engine (UDH_NUMERIC_FP32, csrc/cnn_simt.cu) against float64 and against its own restated arithmetic,
on its own gates, at the step's batch sizes and at a 256-pixel patch.

The two-limb backward is certified against this engine's backward on the same forward state (test_gpu_full_batch.py), so
this engine is the anchor of that chain, and it is the only mode for patches above 128.  Its kernels are fixed fp32
sequences (oracle/simt_fp32.py), so each layer kernel gets three checks at every instance the step launches (conv1_1 two
planes; conv1_2; conv2_x; conv3_1; conv3_2; conv4_x; the dgrad of every layer but conv1_1, with the fused ReLU mask where the
layer below is not a pool; the weight gradients; pool1-3), at B in {1, 3, 128, 129} (P = 128) and {1, 8} (P = 256):
  * exact operands: integer x, w, g in -2..2 and integer biases keep every partial sum below 2^24 in any order, so forward,
    dgrad, dW and db equal float64 exactly, atomics included: a lost, doubled or misplaced tile, halo row or channel chunk
    shows with zero tolerance;
  * restated chain: forward and dgrad equal `conv_chain` bit for bit (a corner 8x16 tile of the first and of the last image
    at 16 channels, plus 2048 random elements; every output of both images where that is cheap); dW / db lie within
    gamma_{m-1} sum|p| of the float64 sum of their m restated thread partials (B in {1, 3} at P = 128, B = 1 at P = 256, and
    two elements per layer at B = 128);
  * float64 on every element: |out - ref| <= gamma_{K+1} (sum|x w| + |b|), K = 9 C_in, and for the weight gradients
    gamma_{L+m-1} sum|x g| with L the longest thread chain and m the partials of the reported partition.
The pools equal the routing rule bit for bit on windows of 2, 3 and 4 equal maxima, all-zero windows and +-0, and on the
engine's own post-ReLU activations of images with flat regions.  The whole engine is then checked layer by layer against
float64 applied to its own input activations, its backward (udh_cnn_bwd with a chosen dh4p) against a float64 backward on
its own gates (ReLU masks, pool routing, dropout masks), and one h_loss and one l1_loss step at P = 256 against the oracle.
Each test prints its measured error next to the bound it asserts."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import oracle as O                                               # noqa: E402
from oracle import simt_fp32 as S                                            # noqa: E402
from _pool_ties import tie_windows                                           # noqa: E402
from _fp32_simt import (CONVS, DGRADS, POOLS, P_, acts as _acts, check_bound, check_chain, check_exact,  # noqa: E402
                        check_partials, check_pool, cnn_fwd as _cnn_fwd, conv_bound, conv_params, flat_batch as _flat_batch,
                        image_size, int_tensor as _int_tensor, layer_input as _layer_input, ref_conv, ref_wgrad,
                        simt_conv, simt_wgrad)


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


BATCHES = [(1, 128), (3, 128), (128, 128), (129, 128), (1, 256), (8, 256)]
RESTATE_WGRAD = {(1, 128): 6, (3, 128): 6, (1, 256): 6, (128, 128): 2}     # (B, P) -> dW elements restated per layer
# per-tensor relative L2 of the engine's backward against float64 on its own gates: measured <= 1.74e-6 (B = 129, P = 128) on
# one H100 80 GB HBM3 (700 W power limit), run-to-run difference <= 1.0e-6; bound 5e-6, 2.9x above that and 40x below the 2e-4
# the two-limb backward is held to against this engine
FP32_BWD_BOUND = 5e-6


def _ids(v):
    return "B%d-P%d" % v


# ------------------------------------------------------------------------------------------------ 1. conv forward
@pytest.mark.parametrize("name,div,cin,cout", CONVS)
@pytest.mark.parametrize("BP", BATCHES, ids=_ids)
def test_conv_forward_exact_restated_and_fp64(udh, BP, name, div, cin, cout):
    B, Pz = BP
    H = Pz // div
    seed = B * 1000 + Pz + H + cin
    two = cin == 2
    g = torch.Generator(device="cuda").manual_seed(seed)
    what = "fp32 %s forward B=%d P=%d" % (name, B, Pz)
    # exact operands
    x = _int_tensor(g, (B, H, H, cin)); w = _int_tensor(g, (3, 3, cin, cout)); b = _int_tensor(g, (cout,), -3, 3)
    x1, x2 = (x[..., :1].contiguous(), x[..., 1:].contiguous()) if two else (x, None)
    check_exact(simt_conv(udh, x1, w, b, relu=1, x2=x2), F.relu(ref_conv(x, w, b)), what + " (exact operands)")
    # real values: restated chain and float64 bound
    x = torch.randn(B, H, H, cin, device="cuda", generator=g)
    w = (torch.randn(3, 3, cin, cout, device="cuda", generator=g) / (3 * cin ** 0.5)).contiguous()
    b = (torch.randn(cout, device="cuda", generator=g) * 0.1).contiguous()
    x1, x2 = (x[..., :1].contiguous(), x[..., 1:].contiguous()) if two else (x, None)
    for relu in (1, 0):
        out = simt_conv(udh, x1, w, b, relu=relu, x2=x2)
        n = check_chain(out, x1, w, b, None, relu, False, seed + relu, what + (" relu" if relu else " linear"), x2=x2)
        ref = ref_conv(x, w, b)
        frac = check_bound(out, F.relu(ref) if relu else ref, conv_bound(x, w, b, False), what)
        print("%s relu=%d: exact operands equal, %d restated chains equal, max err %.3f of gamma_{K+1} bound"
              % (what, relu, n, frac))


# ------------------------------------------------------------------------------------------------ 2. dgrad
@pytest.mark.parametrize("name,div,cin,cout,masked", DGRADS)
@pytest.mark.parametrize("BP", BATCHES, ids=_ids)
def test_dgrad_exact_restated_and_fp64(udh, BP, name, div, cin, cout, masked):
    B, Pz = BP
    H = Pz // div
    seed = B * 1000 + Pz + H + cin + 7 * masked
    gen = torch.Generator(device="cuda").manual_seed(seed)
    what = "fp32 %s dgrad%s B=%d P=%d" % (name, " + mask" if masked else "", B, Pz)
    gi = _int_tensor(gen, (B, H, H, cout)); w = _int_tensor(gen, (3, 3, cin, cout))
    mask = _int_tensor(gen, (B, H, H, cin), -1, 2) if masked else None
    ref = ref_conv(gi, w, None, True)
    check_exact(simt_conv(udh, gi, w, mask=mask, dgrad=1), ref * (mask > 0) if masked else ref, what + " (exact operands)")
    gi = (torch.randn(B, H, H, cout, device="cuda", generator=gen) * 0.1).contiguous()
    w = (torch.randn(3, 3, cin, cout, device="cuda", generator=gen) / (3 * cin ** 0.5)).contiguous()
    mask = F.relu(torch.randn(B, H, H, cin, device="cuda", generator=gen)).contiguous() if masked else None
    out = simt_conv(udh, gi, w, mask=mask, dgrad=1)
    n = check_chain(out, gi, w, None, mask, False, True, seed, what)
    ref = ref_conv(gi, w, None, True)
    bound = conv_bound(gi, w, None, True)
    if masked:
        assert (out[mask <= 0] == 0).all(), what
        ref, bound = ref * (mask > 0), bound * (mask > 0)
    frac = check_bound(out, ref, bound, what)
    print("%s: exact operands equal, %d restated chains equal, max err %.3f of gamma_{K+1} bound" % (what, n, frac))


# ------------------------------------------------------------------------------------------------ 3. weight gradients
@pytest.mark.parametrize("name,div,cin,cout", CONVS)
@pytest.mark.parametrize("BP", BATCHES, ids=_ids)
def test_wgrad_exact_partials_and_fp64(udh, BP, name, div, cin, cout):
    B, Pz = BP
    H = Pz // div
    seed = B * 77 + Pz + H + cin
    gen = torch.Generator(device="cuda").manual_seed(seed)
    two = cin == 2
    what = "fp32 %s wgrad B=%d P=%d" % (name, B, Pz)
    split = lambda x: (x[..., :1].contiguous(), x[..., 1:].contiguous()) if two else (x, None)
    x = _int_tensor(gen, (B, H, H, cin)); go = _int_tensor(gen, (B, H, H, cout))
    x1, x2 = split(x)
    dW, db, part = simt_wgrad(udh, x1, go, cin, x2=x2)
    rW, rb = ref_wgrad(x, go)
    assert rW.abs().sum(dim=(0, 1)).max() < 2 ** 24 and go.abs().sum(dim=(0, 1, 2)).max() < 2 ** 24     # stays exact
    check_exact(dW, rW, what + " dW (exact operands)", "ky,kx,ci,co")
    check_exact(db, rb, what + " db (exact operands)", "co")
    ctas, per, rs = part
    tiles = B * (H // 8) * (H // 16)
    assert ctas * per >= tiles > (ctas - 1) * per, part                # the partition covers every tile once
    x = torch.randn(B, H, H, cin, device="cuda", generator=gen)
    go = (torch.randn(B, H, H, cout, device="cuda", generator=gen) * 0.1).contiguous()
    x1, x2 = split(x)
    dW, db, part = simt_wgrad(udh, x1, go, cin, x2=x2)
    rW, rb = ref_wgrad(x, go)
    L, m = per * (8 // rs) * 16, ctas * rs
    g_ = float(S.gamma(L + m - 1))
    fW = check_bound(dW, rW, g_ * ref_wgrad(x.abs(), go.abs())[0], what + " dW", "ky,kx,ci,co")
    fb = check_bound(db, rb, g_ * go.double().abs().sum(dim=(0, 1, 2)), what + " db", "co")
    msg = ""
    if (B, Pz) in RESTATE_WGRAD:
        fp = check_partials(dW, db, x1, go, part, RESTATE_WGRAD[(B, Pz)], seed, what, x2=x2)
        msg = ", %d elements within %.3f of gamma_{m-1} sum|p| of their %d restated partials" % (RESTATE_WGRAD[(B, Pz)], fp, m)
    print("%s: partition %d CTAs x %d tiles x %d row phases; exact operands equal; dW %.3f, db %.3f of gamma_{L+m-1} bound%s"
          % (what, ctas, per, rs, fW, fb, msg))


# ------------------------------------------------------------------------------------------------ 4. pools
@pytest.mark.parametrize("name,div,C", POOLS)
@pytest.mark.parametrize("BP", BATCHES, ids=_ids)
def test_pool_routing_rule_on_ties(udh, BP, name, div, C):
    B, Pz = BP
    H = Pz // div
    gen = torch.Generator(device="cuda").manual_seed(B * 31 + H + C)
    x = tie_windows(gen, B, H, H, C)
    dout = torch.randn(B, H // 2, H // 2, C, device="cuda", generator=gen)
    dout[..., 0] = -0.0                                    # a negative-zero gradient is routed as itself
    ties, zeros = check_pool(udh, x, dout, "fp32 %s B=%d P=%d" % (name, B, Pz))
    windows = B * (H // 2) ** 2 * C
    assert ties > windows // 3 and zeros > windows // 10, (ties, zeros, windows)
    print("fp32 %s B=%d P=%d: forward and routing bit-identical to the rule on %d windows (%d tied positive maxima, %d zero)"
          % (name, B, Pz, windows, ties, zeros))


# ------------------------------------------------------------------------------------------------ 5. whole engine
def _engine(udh, B, Pz, seed, **kw):
    h, w = image_size(Pz)
    eng = udh.engine.HomographyEngine(B, patch_size=Pz, img_h=h, img_w=w, numeric="fp32", seed=None, **kw)
    flat = udh.params.init_flat_large(seed, Pz)
    eng.load_flat(flat)
    return eng, flat


def _conv_params(udh, eng, i, dtype=None):
    return conv_params(eng, i, dtype)


@pytest.mark.parametrize("BP", [(128, 128), (8, 256)], ids=_ids)
def test_engine_forward_layer_by_layer_on_its_own_inputs(udh, BP):
    """Every conv activation of the engine against float64 applied to the engine's own input activation of that layer
    (per-element gamma_{K+1} bound), and every pool bit-identical to the rule on the engine's pre-pool activation, on images
    with flat regions; plus the pool backward kernel on those activations."""
    B, Pz = BP
    eng, _ = _engine(udh, B, Pz, 2)
    batch = _flat_batch(2, B, Pz)
    I1, I2 = batch["I1_aug"].cuda().contiguous(), batch["I2_aug"].cuda().contiguous()
    _cnn_fwd(udh, eng, I1, I2, False, 0)
    acts = _acts(eng)
    report = []
    for i in range(8):
        w, b = _conv_params(udh, eng, i)
        x = _layer_input(acts, I1, I2, i)
        frac = check_bound(acts[i], F.relu(ref_conv(x, w, b)), conv_bound(x, w, b, False), "engine B=%d P=%d layer %d" % (B, Pz, i))
        report.append("conv%d %.3f" % (i, frac))
    gen = torch.Generator(device="cuda").manual_seed(B + Pz)
    for pi, src in ((8, 1), (9, 3), (10, 5)):
        check_exact(acts[pi], S.pool_fwd(acts[src]).double(), "engine B=%d P=%d pool%d" % (B, Pz, pi - 7))
        dout = torch.randn(acts[pi].shape, device="cuda", generator=gen)
        ties, zeros = check_pool(udh, acts[src].contiguous(), dout, "engine B=%d P=%d pool%d" % (B, Pz, pi - 7))
        assert ties > 0 and zeros > 0, (pi, ties, zeros)
        report.append("pool%d exact (%d tied positive maxima, %d zero windows)" % (pi - 7, ties, zeros))
    print("engine forward B=%d P=%d, fraction of the float64 bound: %s" % (B, Pz, ", ".join(report)))


def fp64_backward(udh, eng, acts, I1, I2, dh4p):
    """The engine's backward in float64 on its own gates: ReLU masks from its activations, pool routing by the rule on its
    pre-pool activations, its dropout masks, and its own activations as the weight gradients' inputs."""
    p = {k: v.double() for k, v in eng.named_parameters().items()}
    names = list(p)
    B = eng.B
    m1, m2 = (m.double() for m in eng.dropout_masks())
    a = {k: v.double() for k, v in acts.items()}
    grads = {}
    fc1d = a[11] * m2 * 2
    a4d = (a[7] * m1 * 2).reshape(B, -1)
    grads[names[18]], grads[names[19]] = fc1d.t() @ dh4p, dh4p.sum(0)
    dfc1 = (dh4p @ p[names[18]].t()) * m2 * 2 * (a[11] > 0)
    grads[names[16]], grads[names[17]] = a4d.t() @ dfc1, dfc1.sum(0)
    g = (dfc1 @ p[names[16]].t()).reshape(a[7].shape) * m1 * 2 * (a[7] > 0)
    for i in range(7, -1, -1):
        x = _layer_input(a, I1.double(), I2.double(), i)
        grads[names[2 * i]], grads[names[2 * i + 1]] = ref_wgrad(x, g)
        if i == 0:
            break
        d = ref_conv(g, p[names[2 * i]], None, True)
        g = S.pool_bwd(a[i - 1], d) if i in (2, 4, 6) else d * (a[i - 1] > 0)
    return grads


@pytest.mark.parametrize("BP", [(128, 128), (129, 128), (8, 256)], ids=_ids)
def test_engine_backward_vs_fp64_on_its_own_gates(udh, BP):
    """udh_cnn_bwd after a train-mode forward, with a chosen dh4p, against fp64_backward: every parameter gradient within
    FP32_BWD_BOUND relative L2, twice (the weight gradients' atomics reorder between runs: the difference between the runs is
    reported, not asserted).  The two-limb backward is held to 2e-4 against this engine (test_gpu_full_batch.py), so this
    bound must stay at least 10x below that for the engine to be a sound reference."""
    assert FP32_BWD_BOUND * 10 <= 2e-4
    B, Pz = BP
    eng, _ = _engine(udh, B, Pz, 1)
    batch = _flat_batch(1, min(B, 128), Pz)
    if B > 128:
        idx = torch.arange(B) % 128
        batch = {k: (v[idx] if isinstance(v, torch.Tensor) and v.dim() > 0 and v.shape[0] == 128 else v) for k, v in batch.items()}
    I1, I2 = batch["I1_aug"].cuda().contiguous(), batch["I2_aug"].cuda().contiguous()
    _cnn_fwd(udh, eng, I1, I2, True, 0xC0FFEE + B)
    acts = _acts(eng)
    dh4p = torch.randn(B, 8, device="cuda", generator=torch.Generator(device="cuda").manual_seed(B)).contiguous()
    ref = fp64_backward(udh, eng, acts, I1, I2, dh4p.double())
    runs = []
    for _ in range(2):
        eng.grads.zero_()
        udh.lib.check(udh.L.udh_cnn_bwd(P_(eng.params), P_(I1), P_(I2), P_(dh4p), P_(eng.grads), P_(eng.ws), eng.ws_bytes, B, Pz, 1,
                                        udh.lib.NUMERIC_FP32, None), "udh_cnn_bwd")
        torch.cuda.synchronize()
        runs.append({k: v.clone() for k, v in eng.named_gradients().items()})
    bad, lines, worst = [], [], 0.0
    for name, r in ref.items():
        e = [((run[name].double() - r).norm() / r.norm().clamp_min(1e-300)).item() for run in runs]
        rep = ((runs[0][name].double() - runs[1][name].double()).norm() / r.norm().clamp_min(1e-300)).item()
        worst = max(worst, *e)
        lines.append("  %-34s rel L2 vs fp64 %.2e / %.2e, run to run %.2e" % (name, e[0], e[1], rep))
        if max(e) > FP32_BWD_BOUND:
            bad.append((name, e))
    print("engine backward B=%d P=%d vs fp64 on its own gates (bound %.0e), worst %.2e:\n%s" % (B, Pz, FP32_BWD_BOUND, worst,
                                                                                              "\n".join(lines)))
    assert not bad, bad


def rel_l2(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).norm() / max(b.norm().item(), 1e-30)).item()


@pytest.mark.parametrize("loss_type,lr", [("h_loss", 5e-4), ("l1_loss", 1e-4)])
def test_train_step_P256_vs_oracle(udh, loss_type, lr):
    """One step at a 256-pixel patch (360 x 480 images) against O.train_step with the engine's dropout masks: pred_h4p within
    1e-5 relative, gradients at test_gpu_parity.py's flip-limited level."""
    seed, B, Pz = 0, 2, 256
    specs = udh.params.param_specs(Pz)
    eng, flat = _engine(udh, B, Pz, seed, loss_type=loss_type, lr=lr)
    batch = O.make_batch(seed, B, img_h=360, img_w=480, patch=Pz)
    db = {k: (v.cuda().contiguous() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}
    out = eng.forward(db, train=True)
    keep = tuple(m.cpu().float() for m in eng.dropout_masks())
    eng.backward(db, out)
    flat_t = torch.tensor(flat)
    _, _, _, ref_out, g = O.train_step(flat_t, torch.zeros_like(flat_t), torch.zeros_like(flat_t), 0, batch, specs,
                                       loss_type=loss_type, lr=lr, keep_masks=keep)
    scale = ref_out["pred_h4p"].abs().max().item()
    e = np.abs(out["pred_h4p"].cpu().numpy() - ref_out["pred_h4p"].numpy()).max() / scale
    assert scale > 10.0 and e <= 1e-5, (scale, e)
    got = eng.grads.cpu()
    errs = {name: rel_l2(got[s.offset:s.offset + s.size], g[s.offset:s.offset + s.size]) for name, s in specs.items()}
    print("P=256 %s: pred_h4p rel err %.2e (max |pred_h4p| %.1f px), worst gradient rel L2 %.2e (%s)"
          % (loss_type, e, scale, max(errs.values()), max(errs, key=errs.get)))
    tol = 1e-2 if loss_type == "h_loss" else 2e-2
    assert all(v < tol for v in errs.values()), errs
