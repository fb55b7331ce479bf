"""GPU tests of the fully connected head (fc1: 32768 -> 1024, fc2: 1024 -> 8) against float64 torch on the GPU, element by element.

fc1 holds 33.6 M of the 34.2 M parameters and runs the largest GEMMs of the step, so a per-tensor relative L2 bound is blind
to an error confined to one region of it (one 128-row band of the weight gradient is 4 of its 1024 output tiles).  Here:
  * fc1's three GEMMs (forward y = x.W, weight gradient dW = x^T.dy, data gradient dx = dy.W^T) through udh_debug_fc1, which
    makes exactly the calls of the step, in every numeric mode, at every batch size from 1 to 512 that changes a tile or
    split boundary: y and dx checked per row (image), dW per 128 x 256 output tile of the tensor-core GEMM;
  * row invariance and determinism: a row of y / dx computed inside a large batch is bit-identical to the same row computed
    alone, and two calls are bit-identical;
  * the head inside the step (h_loss, train mode): pred_h4p, the h_loss gradient, fc2's weight / bias gradients, fc1's bias
    and weight gradients, recomputed in float64 from the engine's own conv4_2 output, dropout masks and ReLU gate;
  * the fc1 weight mirror Adam writes equals, bit for bit, the one the forward casts from the updated weights.
Each test prints its measured error next to the bound it asserts."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as O                                               # noqa: E402

F_IN, N_OUT = 32768, 1024
# one full and one partial 64-row k-block / 128-row M tile on each side of 64 and 128, the fp32 mode's split switch
# (B <= 256: 16 splits, 4 beyond), and the largest batch the step is run at
BATCHES = [1, 2, 63, 64, 65, 127, 128, 129, 200, 256, 257, 512]
MODES = ["bf16x3", "bf16", "fp32"]

# max |err| / max |ref| per row (y, dx) and per 128 x 256 tile (dW), set at about twice the worst value measured on an H100
# SXM over all batch sizes and both operand sets; bf16 is measured on bf16-rounded operands (accumulation only)
# (measured worst: two-limb y 8.4e-6, dx 8.5e-6, dW 2.2e-5; bf16 1.6e-6, 2.1e-6, 2.8e-7; fp32 3.8e-6, 2.1e-6, 3.8e-7).  The
# two-limb dW bound is the mode's 3e-5, not twice its worst: at B = 1, 2 an element of dW is one or two products x . dy, and
# each product carries the limb split's own error (up to 3 x 2^-16 of |x dy|: the dropped lo.lo term and the rounding of both
# lo limbs) with no sum over the batch to average it.
BOUND = {
    "bf16x3": dict(y=2e-5, dx=2e-5, dW=3e-5),
    "bf16": dict(y=3e-6, dx=4e-6, dW=6e-7),
    "fp32": dict(y=8e-6, dx=5e-6, dW=8e-7),
}


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
    ns.code = {"bf16x3": _lib.NUMERIC_BF16X3, "bf16": _lib.NUMERIC_BF16, "fp32": _lib.NUMERIC_FP32}
    yield ns
    torch.cuda.empty_cache()


P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None


@pytest.fixture(scope="module")
def weights(udh):
    """fc1's weights [32768, 1024] in fp32 and as the float64 reference, plain and bf16-rounded."""
    g = torch.Generator(device="cuda").manual_seed(11)
    w = (torch.randn(F_IN, N_OUT, device="cuda", generator=g) * 0.01).contiguous()
    wb = w.bfloat16().float()
    return {False: (w, w.double()), True: (wb, wb.double())}


def _operands(kind, B, round_bf16):
    """x [B, F], dy [B, 1024] in fp32.
    step: x post-ReLU with conv4_2's dropout applied (x2 or 0), dy with the dropout / ReLU zeros of dfc1 and the 1/B of the
          batch mean;
    dense: randn, dy row b scaled by 10^(-8 + 7 b / (B - 1)): the gradients of a step span that range."""
    g = torch.Generator(device="cuda").manual_seed(1000 * B + (1 if kind == "step" else 2))
    x = torch.randn(B, F_IN, device="cuda", generator=g)
    dy = torch.randn(B, N_OUT, device="cuda", generator=g)
    if kind == "step":
        x = x.clamp_min(0) * (torch.rand(B, F_IN, device="cuda", generator=g) < 0.5) * 2.0
        dy = dy * (torch.rand(B, N_OUT, device="cuda", generator=g) < 0.25) * 2.0 / B
    else:
        dy = dy * torch.logspace(-8, -1, B, device="cuda")[:, None]
    if round_bf16:
        x, dy = x.bfloat16().float(), dy.bfloat16().float()
    return x.contiguous(), dy.contiguous()


def _fc1(udh, mode, x, w, dy=None):
    """udh_debug_fc1 -> y, dW, dx, scratch.  Outputs start as NaN (dW as 0 in the fp32 mode, which accumulates it), so an
    element a kernel never writes fails the check."""
    B = x.shape[0]
    nan = float("nan")
    y = torch.full((B, N_OUT), nan, device="cuda")
    dW = dx = None
    if dy is not None:
        dW = torch.zeros(F_IN, N_OUT, device="cuda") if mode == "fp32" else torch.full((F_IN, N_OUT), nan, device="cuda")
        dx = torch.full((B, F_IN), nan, device="cuda")
    n = udh.L.udh_debug_fc1_scratch_bytes(B, udh.code[mode])
    assert (n > 0) == (mode != "fp32")
    scratch = torch.empty(n, device="cuda", dtype=torch.uint8) if n else None
    rc = udh.L.udh_debug_fc1(udh.code[mode], P(x), P(w), P(dy), P(y), P(dW), P(dx), P(scratch), B, None)
    assert rc == 0, udh.L.udh_last_error()
    torch.cuda.synchronize()
    return y, dW, dx, scratch


def _check_rows(got, ref, tol, what):
    """max |got - ref| against the tensor's max |ref| and, per row (image), against that row's max |ref|.
    Returns (tensor error, worst row error); the failure message names the rows."""
    assert torch.isfinite(got).all(), "%s: non-finite output" % what
    d = (got.double() - ref).abs()
    err = (d.max() / ref.abs().max()).item()
    rel = d.amax(dim=1) / ref.abs().amax(dim=1).clamp_min(1e-300)
    worst = rel.max().item()
    bad = (rel > tol).nonzero().flatten().tolist()
    msg = "; ".join("image %d (rel err %.2e)" % (b, rel[b].item()) for b in bad[:6])
    assert err <= tol and not bad, "%s: max rel err %.2e, worst image %.2e > %.0e; %d images fail: %s" % (what, err, worst, tol, len(bad), msg)
    return err, worst


def _check_tiles(got, ref, tol, what):
    """dW [32768, 1024] per 128 x 256 output tile (mt, nt) of the tensor-core GEMM, against the tile's max |ref|."""
    assert torch.isfinite(got).all(), "%s: non-finite output" % what
    d = (got.double() - ref).abs()
    err = (d.max() / ref.abs().max()).item()
    td = d.view(F_IN // 128, 128, N_OUT // 256, 256).amax(dim=(1, 3))
    del d
    rel = td / ref.abs().view(F_IN // 128, 128, N_OUT // 256, 256).amax(dim=(1, 3)).clamp_min(1e-300)
    worst = rel.max().item()
    bad = (rel > tol).nonzero().tolist()
    msg = "; ".join("tile (mt %d, nt %d) rel err %.2e" % (mt, nt, rel[mt, nt].item()) for mt, nt in bad[:6])
    assert err <= tol and not bad, "%s: max rel err %.2e, worst tile %.2e > %.0e; %d tiles fail: %s" % (what, err, worst, tol, len(bad), msg)
    return err, worst


# ------------------------------------------------------------------------------------------------ a-c. fc1's GEMMs vs fp64
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("kind", ["step", "dense"])
@pytest.mark.parametrize("mode", MODES)
def test_fc1_gemms_vs_fp64(udh, weights, mode, kind, B):
    """y = x.W, dW = x^T.dy and dx = dy.W^T of udh_debug_fc1 against float64.  The single-pass bf16 mode gets bf16-rounded
    operands, so only its accumulation is measured."""
    rb = mode == "bf16"
    w, w64 = weights[rb]
    x, dy = _operands(kind, B, rb)
    y, dW, dx, _ = _fc1(udh, mode, x, w, dy)
    x64, dy64 = x.double(), dy.double()
    tol = BOUND[mode]
    what = "%s %s B=%d" % (mode, kind, B)
    ey = _check_rows(y, x64 @ w64, tol["y"], what + " y")
    ex = _check_rows(dx, dy64 @ w64.T, tol["dx"], what + " dx")
    del dx
    eW = _check_tiles(dW, x64.T @ dy64, tol["dW"], what + " dW")
    print("fc1 %-6s %-5s B=%3d: y %.2e (worst image %.2e), dx %.2e (worst image %.2e), dW %.2e (worst tile %.2e); bounds %.0e %.0e %.0e"
          % (mode, kind, B, ey[0], ey[1], ex[0], ex[1], eW[0], eW[1], tol["y"], tol["dx"], tol["dW"]))


# ------------------------------------------------------------------------------------------------ d. invariance, determinism
@pytest.mark.parametrize("B", [129, 512])
@pytest.mark.parametrize("mode", MODES)
def test_fc1_rows_invariant_to_batch_and_deterministic(udh, weights, mode, B):
    """Two calls give bit-identical y, dW and dx.  A row of y / dx sums the same chain of k-blocks whatever M tile it sits
    in, and the tensor-core split count depends only on the feature count: so rows at B = 129 / 512 equal, bit for bit, the
    same rows computed alone at B = 1 (first and last rows of M tiles, the one-row tail).  The fp32 mode's split count
    changes above B = 256: there the forward rows agree within the fc1 bound only."""
    rb = mode == "bf16"
    w, _ = weights[rb]
    x, dy = _operands("dense", B, rb)
    y, dW, dx, _ = _fc1(udh, mode, x, w, dy)
    y2, dW2, dx2, _ = _fc1(udh, mode, x, w, dy)
    assert torch.equal(y, y2) and torch.equal(dW, dW2) and torch.equal(dx, dx2), "%s B=%d: two calls differ" % (mode, B)
    del dW, dW2, y2, dx2
    rows = sorted({0, 1, 63, 64, 127, 128, B - 1})
    exact_y = mode != "fp32" or B <= 256
    worst = 0.0
    for r in rows:
        y1, _, dx1, _ = _fc1(udh, mode, x[r:r + 1].contiguous(), w, dy[r:r + 1].contiguous())
        assert torch.equal(dx1[0], dx[r]), "%s B=%d: dx row %d differs from the same row computed alone" % (mode, B, r)
        if exact_y:
            assert torch.equal(y1[0], y[r]), "%s B=%d: y row %d differs from the same row computed alone" % (mode, B, r)
        else:
            e = ((y1[0] - y[r]).abs().max() / y1[0].abs().max()).item()
            worst = max(worst, e)
            assert e <= BOUND[mode]["y"], (mode, B, r, e)
    print("fc1 %-6s B=%3d: bit-identical on repeat; rows %s of dx bit-identical to B = 1, of y %s"
          % (mode, B, rows, "bit-identical" if exact_y else "within %.2e (bound %.0e)" % (worst, BOUND[mode]["y"])))


# ------------------------------------------------------------------------------------------------ e. the head inside the step
_BATCH = {}


def _batch(B):
    """O.make_batch(7, 128), rows repeated to B."""
    if 128 not in _BATCH:
        _BATCH[128] = O.make_batch(7, 128)
    b = _BATCH[128]
    idx = torch.arange(B) % 128
    return {k: (v[idx].cuda().contiguous() if isinstance(v, torch.Tensor) and v.dim() > 0 and v.shape[0] == 128 else v)
            for k, v in b.items()}


def _fp32_chain(a, b):
    """a [M, K] . b[N, K]^T as the CUDA-core sgemm computes it for small K: one fp32 fma chain per element, k in order
    (each fp32 x fp32 product is exact in float64, so float64 add + fp32 rounding is the fma)."""
    acc = torch.zeros(a.shape[0], b.shape[0], device=a.device, dtype=torch.float32)
    for k in range(a.shape[1]):
        acc = (acc.double() + a[:, k:k + 1].double() * b[:, k].double()[None, :]).float()
    return acc


# relative to the tensor's max |ref| (fc1's weight gradient: to its tile's), about twice the worst of B = 128, 129 on an H100
HEAD_BOUND = {
    "bf16x3": dict(pred=1e-5, dh4p=3e-7, dW2=8e-7, db2=2e-7, db1=2e-7, dW1=1e-5),
    "bf16": dict(pred=8e-7, dh4p=3e-7, dW2=8e-7, db2=2e-7, db1=2e-7, dW1=3e-7),
    "fp32": dict(pred=8e-7, dh4p=3e-7, dW2=5e-7, db2=2e-7, db1=3e-7, dW1=6e-7),
}


@pytest.mark.parametrize("B", [128, 129])
@pytest.mark.parametrize("mode", MODES)
def test_head_in_step_vs_fp64(udh, mode, B):
    """The head of an h_loss train-mode step (udh_cnn_fwd, h4p loss, udh_cnn_bwd) recomputed in float64 from the engine's own
    conv4_2 output, dropout masks and fc1 ReLU gate, so no gate can flip and every bound is the kernels' own.  Each gradient
    is recomputed from the engine's inputs to that kernel (its dh4p, its fc1 activation), so each comparison measures one
    kernel.  Also: the BWD_HEAD + BWD_CONVS phases of the data-parallel path leave the same fc gradients bit for bit (the
    fp32 mode's conv weight gradients are atomic sums, so the conv slice is not compared)."""
    L, lib = udh.L, udh.lib
    flat = udh.params.init_flat_large(8)
    db = _batch(B)
    e = udh.engine.HomographyEngine(B, seed=None, numeric=mode, loss_type="h_loss", lr=5e-4); e.load_flat(flat)
    out = e.forward(db, train=True, dropout_seed=99)
    e.backward(db, out)
    torch.cuda.synchronize()
    grads = e.grads.clone()
    g2 = torch.zeros_like(e.grads)
    args = (e._p(e.params), e._p(db["I1_aug"]), e._p(db["I2_aug"]), e._p(out["_dh4p"]), e._p(g2), e._p(e.ws), e.ws_bytes, B, e.Pz, 1,
            e.numeric)
    lib.check(L.udh_cnn_bwd_phase(*args, lib.BWD_HEAD, udh.ops._stream()), "udh_cnn_bwd_phase(head)")
    lib.check(L.udh_cnn_bwd_phase(*args, lib.BWD_CONVS, udh.ops._stream()), "udh_cnn_bwd_phase(convs)")
    torch.cuda.synchronize()
    head, _ = udh.engine.dp_slices(udh.params.param_specs())
    assert torch.equal(g2[head], grads[head]), "%s B=%d: BWD_HEAD + BWD_CONVS leaves other fc gradients than udh_cnn_bwd" % (mode, B)
    del g2

    specs = udh.params.param_specs()
    p = {n: e.params[s.offset:s.offset + s.size].reshape(s.shape) for n, s in specs.items()}
    gr = {n: grads[s.offset:s.offset + s.size].reshape(s.shape) for n, s in specs.items()}
    W1, b1 = p["model/fc1/fc1/weights"], p["model/fc1/fc1/biases"].double()
    W2, b2 = p["model/fc2/fc2/weights"], p["model/fc2/fc2/biases"].double()
    m1, m2 = e.dropout_masks()
    keep1, keep2 = m1.reshape(B, F_IN).double() * 2.0, m2.double() * 2.0
    x = e.activation(7).reshape(B, F_IN)                       # conv4_2, NHWC flatten (slim.flatten)
    act11 = e.activation(11).reshape(B, N_OUT)                 # fc1 after ReLU, before dropout
    gate = (act11 > 0).double()
    xd = x.double() * keep1
    dh4p = out["_dh4p"]
    pred = out["pred_h4p"]
    gt = db["gt"].double()
    if mode == "bf16":                                          # the mode's fc1 operands: bf16 copies, fp32 accumulation
        xd, W1_64 = xd.bfloat16().double(), W1.bfloat16().double()
    else:
        W1_64 = W1.double()
    # forward: pred_h4p from the engine's conv4_2 output and gates
    pred_ref = ((xd @ W1_64 + b1) * gate * keep2) @ W2.double() + b2
    # h_loss gradient from the engine's pred (h4p_loss_kernel alone)
    d = pred.double() - gt
    dh4p_ref = d / (8.0 * B * d.square().mean().sqrt())
    # fc2 from the engine's fc1 activation and dh4p
    fc1d = act11.double() * keep2
    dW2_ref = fc1d.T @ dh4p.double()
    db2_ref = dh4p.double().sum(dim=0)
    if mode == "bf16":                                          # dfc1 exactly as the engine forms it, then its bf16 copy
        dfc1 = _fp32_chain(dh4p, W2).double() * keep2 * gate
        db1_ref = dfc1.sum(dim=0)
        dfc1 = dfc1.bfloat16().double()
    else:
        dfc1 = (dh4p.double() @ W2.double().T) * keep2 * gate
        db1_ref = dfc1.sum(dim=0)
    tol = HEAD_BOUND[mode]
    rel = lambda a, b: ((a.double() - b).abs().max() / b.abs().max()).item()
    errs = dict(pred=rel(pred, pred_ref), dh4p=rel(dh4p, dh4p_ref), dW2=rel(gr["model/fc2/fc2/weights"], dW2_ref),
                db2=rel(gr["model/fc2/fc2/biases"], db2_ref), db1=rel(gr["model/fc1/fc1/biases"], db1_ref))
    _, errs["dW1"] = _check_tiles(gr["model/fc1/fc1/weights"], xd.T @ dfc1, tol["dW1"], "%s B=%d fc1 weight gradient in the step" % (mode, B))
    print("head %-6s B=%3d: %s" % (mode, B, ", ".join("%s %.2e (bound %.0e)" % (k, v, tol[k]) for k, v in errs.items())))
    bad = {k: v for k, v in errs.items() if not v <= tol[k]}
    assert not bad, bad
    del e


# ------------------------------------------------------------------------------------------------ f. Adam's weight mirror
@pytest.mark.parametrize("mode", ["bf16x3", "bf16"])
def test_adam_mirror_equals_forward_cast(udh, mode):
    """After a train step the step's next forward trusts the fc1 weight mirror Adam wrote (UDH_FWD_FC1_MIRROR_CURRENT); the
    certification above holds for the step only if that mirror equals, bit for bit, the planes the forward casts from the
    updated fp32 weights: checked against udh_debug_fc1's own cast and against a forward with the mirror marked stale."""
    B = 4
    flat = udh.params.init_flat_large(9)
    db = _batch(B)
    e = udh.engine.HomographyEngine(B, seed=None, numeric=mode, loss_type="h_loss", lr=5e-4); e.load_flat(flat)
    mp, mb, mc, _ = e._mirror
    off = mp - e.ws.data_ptr()
    limbs = 2 if mode == "bf16x3" else 1
    nbytes = 2 * limbs * mc
    e.eval_step(db)                                             # casts the initial weights
    before = e.ws[off:off + nbytes].clone()
    e.train_step(db)
    torch.cuda.synchronize()
    assert e._mirror_is_current()
    adam = e.ws[off:off + nbytes].clone()
    assert not torch.equal(adam, before), "the step left the mirror unchanged"
    w = e.params[mb:mb + mc]
    # udh_debug_fc1 at B = 1 casts w itself; its scratch holds x's copy (32768 x limbs 16-bit values) and then the mirror
    _, _, _, scratch = _fc1(udh, mode, torch.zeros(1, F_IN, device="cuda"), w)
    x_bytes = -(-2 * limbs * F_IN // 256) * 256
    n_diff = (scratch[x_bytes:x_bytes + nbytes] != adam).sum().item()
    assert n_diff == 0, "%s: %d bytes of Adam's mirror differ from the forward's cast of the updated weights" % (mode, n_diff)
    e._mirror_current = False
    e.eval_step(db)                                             # casts the updated weights into the workspace
    torch.cuda.synchronize()
    assert torch.equal(e.ws[off:off + nbytes], adam), "%s: Adam's mirror differs from a stale-mirror forward's cast" % mode
    print("%s: Adam's fc1 mirror (%d planes of %d values) bit-identical to the forward's cast of the updated weights" % (mode, limbs, mc))
    del e
