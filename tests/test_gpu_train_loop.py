"""GPU tests of the train step beyond the first: the state one step hands to the next.

  * the Adam kernel (udh_adam_step_mirror_ex) against float64 element by element, inside oracle.optim.adam_bound, on the
    regimes where the update goes wrong (|g| from 1e-12 to 1e3, t = 1, sqrt(v) ~ eps, m against g, g = m = v = 0), at every
    grad_scale and alpha_t the engine passes, from 4 floats to the whole 34 192 264-float buffer; its guard bands, its
    one- and two-limb fc1 mirror, zero_grad / keep_grad, and bit-identity across grid caps and range splits;
  * the engine's step mapping over 8 steps across bench.py's staircase boundary (step 3 570) and near step 150 000, in all
    three numeric modes: parameters, m and v against float64 Adam from the captured gradient, what the update leaves in the
    gradient buffer, and the mirror;
  * continuation equals resumption: from state_dict, the TF checkpoint and a .pt file, with an eval step in between, and with
    a second engine interleaved; dropout statistics across steps;
  * the overlapped update (UDH_OVERLAP_UPDATE=1) and trainer.HostStepper's two-slot ring against the plain step.
Every bound check prints its worst measured / bound ratio."""
import ctypes
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import optim as Q                                                # noqa: E402

LR, MIN_LR = 5e-4, 0.9e-4            # bench.py's setting: decay_steps = 3570
B = 128
K = 8
START = 3567                         # steps 3567 ... 3574 cross the first staircase boundary
SEED = 1234
WORST = {}


@pytest.fixture(scope="module")
def udh():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from unsuperviseddeephomographyral2018_b200 import _lib, engine, ops, params, synthetic, trainer
    _lib.require_device()

    class NS:
        pass
    ns = NS()
    ns.lib, ns.ops, ns.engine, ns.params, ns.synthetic, ns.trainer, ns.L = _lib, ops, engine, params, synthetic, trainer, _lib.lib
    yield ns
    ns.L.udh_set_adam_grid(0)
    if WORST:
        print("\nworst measured / bound: " + "  ".join("%s %.3f" % kv for kv in sorted(WORST.items())))


def _note(key, r):
    WORST[key] = max(WORST.get(key, 0.0), float(r))
    assert r <= 1.0, (key, float(r))


def ptr(t, off_bytes=0):
    return ctypes.c_void_p(t.data_ptr() + off_bytes)


_BATCHES = {}


def batch(udh, k, rgb=False):
    """Distinct synthetic batch k at B = 128 (device generator)."""
    if (k, rgb) not in _BATCHES:
        b = udh.synthetic.make_batch_fast(B, seed=1000 + k, want_rgb=rgb)
        if rgb:
            b = dict(b, I_aug=b["I_aug_rgb"])
        _BATCHES[(k, rgb)] = {kk: v for kk, v in b.items() if isinstance(v, torch.Tensor)}
    return _BATCHES[(k, rgb)]


def alpha_ref(step):
    """alpha_t of the update from `step`, restated (float64 form, exact beta powers; DESIGN section 2)."""
    t = step + 1
    lr_t = LR * 0.96 ** (step // Q.decay_steps(LR, MIN_LR))
    return lr_t, lr_t * math.sqrt(1.0 - 0.999 ** t) / (1.0 - 0.9 ** t)


def split_ref(p, limbs):
    """The fc1 mirror Adam writes from the new weights p (fp32, device): bf16 round-to-nearest, and for two limbs
    hi = bf16(p), lo = bf16(p - hi) (tc_common.cuh split2), hi plane then lo plane; as int16 words."""
    hi = p.to(torch.bfloat16)
    if limbs == 1:
        return hi.view(torch.int16)
    lo = (p - hi.float()).to(torch.bfloat16)
    return torch.cat([hi.view(torch.int16), lo.view(torch.int16)])


def check_adam(key, p0, g0, m0, v0, p1, m1, v1, alpha, gs=1.0):
    """p1, m1, v1 (kernel) against float64 Adam from p0, g0, m0, v0 within adam_bound; p bit-unchanged where g = m = v = 0."""
    P64, M64, V64 = Q.adam64(p0, g0, m0, v0, alpha, grad_scale=gs)
    ep, em, ev = Q.adam_bound(p0, g0, m0, v0, alpha, grad_scale=gs)
    for name, got, ref, b in (("p", p1, P64, ep), ("m", m1, M64, em), ("v", v1, V64, ev)):
        _note("%s.%s" % (key, name), ((got.double() - ref).abs() / b).max().item())
    z = (g0 == 0) & (m0 == 0) & (v0 == 0)
    assert torch.equal(p1[z], p0[z])


# ------------------------------------------------------------------------------------------------ 2. the Adam kernel
GUARD = 64


def run_adam(udh, p, g, m, v, alpha, gs=1.0, mirror=None, zero_grad=1, segments=None):
    """udh_adam_step_mirror_ex on [0, n) of device copies of p, g, m, v, each between two GUARD-float bands, the pointers at
    float offset GUARD (4-aligned and nonzero, as engine._adam passes them).  mirror = (begin, count, limbs, keep_grad).
    segments: split points of [0, n), one call per piece (the mirror must fall inside one).  Returns the full buffers."""
    n = p.numel()
    sentinel = lambda: torch.full((GUARD,), -7.25, device="cuda")
    bufs = [torch.cat([sentinel(), x.cuda(), sentinel()]).contiguous() for x in (p, g, m, v)]
    mb, mc, limbs, keep = mirror if mirror is not None else (0, 0, 1, 0)
    mir = torch.full((2 * GUARD + limbs * mc,), 0x5A5A, dtype=torch.int16, device="cuda")
    cuts = [0, n] if segments is None else [0] + list(segments) + [n]
    for a, b in zip(cuts[:-1], cuts[1:]):
        inside = mirror is not None and a <= mb and mb + mc <= b
        udh.lib.check(udh.L.udh_adam_step_mirror_ex(*(ptr(t, 4 * (GUARD + a)) for t in bufs), b - a, float(alpha), 0.9, 0.999, 1e-8,
                                                   float(gs), zero_grad, ptr(mir, 2 * GUARD) if inside else None,
                                                   (mb - a) if inside else 0, mc if inside else 0, keep, limbs, udh.ops._stream()),
                      "udh_adam_step_mirror_ex")
    torch.cuda.synchronize()
    return bufs + [mir]


def check_run(key, out, p, g, m, v, alpha, gs, mirror, zero_grad):
    pb, gb, mb_, vb, mir = out
    n = p.numel()
    for t in (pb, gb, mb_, vb):
        assert torch.equal(t[:GUARD], t.new_full((GUARD,), -7.25)) and torch.equal(t[-GUARD:], t.new_full((GUARD,), -7.25))
    pd, gd, md, vd = (x.cuda() for x in (p, g, m, v))
    p1, g1, m1, v1 = (t[GUARD:GUARD + n] for t in (pb, gb, mb_, vb))
    check_adam(key, pd, gd, md, vd, p1, m1, v1, alpha, gs)
    b0, c, limbs, keep = mirror if mirror is not None else (0, 0, 1, 0)
    assert (mir[:GUARD] == 0x5A5A).all() and (mir[GUARD + limbs * c:] == 0x5A5A).all()
    if mirror is not None:
        assert torch.equal(mir[GUARD:GUARD + limbs * c], split_ref(p1[b0:b0 + c], limbs)), "%s: mirror" % key
    if not zero_grad:
        assert torch.equal(g1, gd)
        return
    inside = torch.zeros(n, dtype=torch.bool, device="cuda")
    if mirror is not None and keep:
        inside[b0:b0 + c] = True
    assert torch.equal(g1[inside], gd[inside]) and (g1[~inside] == 0).all()


GS = [1.0, 0.5, 0.125, 1.0 / 3.0]
TS = [1, 2, 10, 3570, 150000]


@pytest.mark.parametrize("n", [4, 36, 4132])
def test_adam_kernel_small_vs_float64(udh, n):
    """Every grad_scale x alpha_t, mirrors of one and two limbs, keep_grad on and off, zero_grad on and off."""
    rng = np.random.default_rng(n)
    for i, (gs, t) in enumerate((gs, t) for gs in GS for t in TS):
        p, g, m, v = (torch.from_numpy(x) for x in Q.adam_inputs(rng, n))
        alpha = np.float32(alpha_ref(t - 1)[1])
        mb = 0 if n == 4 else 4 * (i % 3 + 1)
        mirror = (mb, n - mb - (0 if n == 4 else 8), 1 + i % 2, int(i % 4 != 3))
        zg = int(i % 5 != 4)
        out = run_adam(udh, p, g, m, v, alpha, gs, mirror, zg)
        check_run("adam.n%d" % n, out, p, g, m, v, alpha, gs, mirror, zg)


def test_adam_kernel_whole_buffer_vs_float64(udh):
    """The real flat buffer (34 192 264 parameters, padded to 34 192 288 floats) with fc1's real mirror range, once per limb
    count."""
    specs = udh.params.param_specs()
    n = udh.params.total_floats(specs)
    assert n >= 34192264 and n % 4 == 0
    w = specs["model/fc1/fc1/weights"]
    mirror_at = (w.offset, w.size)
    rng = np.random.default_rng(5)
    p, g, m, v = (torch.from_numpy(x) for x in Q.adam_inputs(rng, n))
    for limbs, gs, t in ((2, 1.0 / 3.0, 1), (1, 1.0, 150000)):
        alpha = np.float32(alpha_ref(t - 1)[1])
        mirror = mirror_at + (limbs, 1)
        out = run_adam(udh, p, g, m, v, alpha, gs, mirror, 1)
        check_run("adam.full", out, p, g, m, v, alpha, gs, mirror, 1)
        del out


def test_adam_kernel_bit_identical_across_grids_and_splits(udh):
    n = 266276
    rng = np.random.default_rng(11)
    p, g, m, v = (torch.from_numpy(x) for x in Q.adam_inputs(rng, n))
    alpha = np.float32(alpha_ref(3569)[1])
    mirror = (1024, 200000, 2, 1)
    ref = run_adam(udh, p, g, m, v, alpha, 0.5, mirror)
    try:
        for grid in (1, 3, 264, 0):
            udh.lib.check(udh.L.udh_set_adam_grid(grid), "udh_set_adam_grid")
            got = run_adam(udh, p, g, m, v, alpha, 0.5, mirror)
            assert all(torch.equal(a, b) for a, b in zip(got, ref)), "grid %d" % grid
    finally:
        udh.L.udh_set_adam_grid(0)
    for seg in ([1024, 201024], [512, 1024, 201024, 230000]):
        got = run_adam(udh, p, g, m, v, alpha, 0.5, mirror, segments=seg)
        assert all(torch.equal(a, b) for a, b in zip(got, ref)), "segments %s" % seg


# ------------------------------------------------------------------------------------------------ 3 / 4. the loop
def make_engine(udh, numeric, loss="h_loss", batch_size=B, flat=None, start=START):
    e = udh.engine.HomographyEngine(batch_size, seed=None, numeric=numeric, loss_type=loss, lr=LR, min_lr=MIN_LR)
    e.load_flat(udh.params.init_flat_large(3) if flat is None else flat)
    e.global_step = start
    e.dropout_seed = SEED
    return e


def step(udh, e, db):
    """train_step with the gradient captured between the backward and the update (engine.train_step's default path)."""
    a = e._fill_args(db, True)
    e._apply_sm_policy()
    udh.lib.check(udh.L.udh_step_forward_backward(ctypes.byref(a), udh.lib.STEP_ALL, udh.ops._stream()), "udh_step_forward_backward")
    out = e._step_out(db)
    m1, m2 = e.dropout_masks()
    res = dict(grads=e.grads.clone(), pred=out["pred_h4p"].clone(), metrics=out["h4p_metrics"].clone(),
               photo=out["photo_losses"].clone(), mask1=m1.clone(), mask2=m2.clone(), step=e.global_step)
    res["lr"] = e.update()
    res.update(params=e.params.clone(), m=e.adam_m.clone(), v=e.adam_v.clone(), grads_after=e.grads.clone(), mirror=mirror_of(e))
    return res


def mirror_of(e):
    if e._mirror is None:
        return None
    mp, mb, mc, _ = e._mirror
    off = mp - e.ws.data_ptr()
    limbs = 2 if e.numeric_name == "bf16x3" else 1
    return e.ws[off:off + 2 * limbs * mc].view(torch.int16).clone()


def snapshot(e):
    return dict(params=e.params.clone(), adam_m=e.adam_m.clone(), adam_v=e.adam_v.clone(), global_step=e.global_step)


BITWISE = ("pred", "metrics", "grads", "params", "m", "v", "mirror", "mask1", "mask2")


def assert_same(a, b, what, keys=BITWISE):
    for k in keys:
        if a[k] is None:
            assert b[k] is None
            continue
        assert torch.equal(a[k], b[k]), "%s: %s differs" % (what, k)


def check_mapping(udh, e, res, prev, key):
    """One step of the loop against float64 Adam, the schedule, the gradient buffer after the update and the mirror."""
    s = res["step"]
    lr_t, alpha = alpha_ref(s)
    assert res["lr"] == lr_t, (s, res["lr"], lr_t)
    check_adam(key, prev["params"], res["grads"], prev["m"], prev["v"], res["params"], res["m"], res["v"], np.float32(alpha))
    if e._mirror is not None:
        _, mb, mc, stored = e._mirror
        assert stored
        kept = torch.zeros_like(res["grads"], dtype=torch.bool)
        kept[mb:mb + mc] = True
        assert torch.equal(res["grads_after"][kept], res["grads"][kept]) and (res["grads_after"][~kept] == 0).all()
        limbs = 2 if e.numeric_name == "bf16x3" else 1
        assert torch.equal(res["mirror"], split_ref(res["params"][mb:mb + mc], limbs)), "step %d: mirror" % s
    else:
        assert (res["grads_after"] == 0).all()


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / max(b.norm().item(), 1e-30)).item()


def worst_grad_rel_l2(udh, a, b):
    return max(rel_l2(a[s.offset:s.offset + s.size], b[s.offset:s.offset + s.size]) for s in udh.params.param_specs().values())


GRAD_ENVELOPE = 1e-4        # per-tensor rel L2 between two runs of a step whose backward accumulates with atomics


@pytest.mark.parametrize("numeric", ["bf16x3", "bf16", "fp32"])
def test_loop_step_mapping_and_resumption(udh, numeric):
    """8 steps from global_step 3567 on distinct batches: each step's update against float64 Adam from the captured gradient
    and alpha_t; after the update fc1's weight gradient is kept (tensor-core modes) and everything else is zero; the mirror is
    the split of the new weights.  Then a fresh engine resumed from the state before step k reproduces step k: bit for bit in
    the tensor-core modes (its fc1 gradient is a store, so a fresh buffer gives the same one), and in fp32, whose backward
    accumulates with atomics, with bit-identical pred_h4p and gradients within GRAD_ENVELOPE."""
    E = make_engine(udh, numeric)
    snaps, runs = [], []
    prev = dict(params=E.params.clone(), m=E.adam_m.clone(), v=E.adam_v.clone())
    for k in range(K):
        snaps.append(snapshot(E))
        res = step(udh, E, batch(udh, k))
        check_mapping(udh, E, res, prev, "loop.%s" % numeric)
        prev = res
        runs.append({kk: res[kk] for kk in BITWISE + ("step",)})
    assert [r["step"] for r in runs] == list(range(START, START + K))
    F = make_engine(udh, numeric, start=0)
    for k in (1, 3, 6):                                   # F reused: load_state_dict must drop F's own current mirror
        F.load_state_dict(snaps[k])
        got = step(udh, F, batch(udh, k))
        if numeric != "fp32":
            assert_same(runs[k], got, "%s resume at step %d" % (numeric, START + k))
        else:
            assert torch.equal(got["pred"], runs[k]["pred"]) and torch.equal(got["mask2"], runs[k]["mask2"])
            r = worst_grad_rel_l2(udh, got["grads"], runs[k]["grads"])
            print("fp32 resume at step %d: worst per-tensor gradient rel L2 %.2e (envelope %.0e)" % (START + k, r, GRAD_ENVELOPE))
            assert r <= GRAD_ENVELOPE
    # dropout: consecutive steps draw independent masks, each keeps half of every sample, conv4 and fc1 masks uncorrelated
    for a, b in zip(runs[:-1], runs[1:]):
        for key in ("mask1", "mask2"):
            x, y = a[key] != 0, b[key] != 0
            N = x.numel()
            agree = (x == y).double().mean().item()
            assert abs(agree - 0.5) <= 5 * 0.5 / math.sqrt(N), (key, agree)
    for r in runs:
        for key in ("mask1", "mask2"):
            x = (r[key] != 0).reshape(B, -1).double()
            rate = x.mean(1)
            assert (rate - 0.5).abs().max().item() <= 5 * 0.5 / math.sqrt(x.shape[1]), key
        # same local element index in both masks: agree on half of them (a shared salt would make them equal)
        x1, x2 = (r["mask1"] != 0).reshape(B, -1)[:, :1024], r["mask2"] != 0
        agree = (x1 == x2).double().mean().item()
        assert abs(agree - 0.5) <= 5 * 0.5 / math.sqrt(x2.numel()), agree
    del E, F
    torch.cuda.empty_cache()


def test_loop_near_the_last_step(udh):
    """Steps 149 996 ... 149 999: alpha_t with both beta powers ~0."""
    E = make_engine(udh, "bf16x3", start=149996)
    prev = dict(params=E.params.clone(), m=E.adam_m.clone(), v=E.adam_v.clone())
    for k in range(4):
        res = step(udh, E, batch(udh, k))
        check_mapping(udh, E, res, prev, "loop.end")
        prev = res
    assert E.global_step == 150000


def test_l1_loss_resumption_within_envelope(udh):
    """l1_loss's photometric sums are fp64 atomics: resuming gives bit-identical pred_h4p, gradients within GRAD_ENVELOPE
    of the continued run, and the same spread as two fresh resumed runs."""
    E = make_engine(udh, "bf16x3", loss="l1_loss")
    step(udh, E, batch(udh, 0))
    snap = snapshot(E)
    ref = step(udh, E, batch(udh, 1))
    got = []
    for _ in range(2):
        F = make_engine(udh, "bf16x3", loss="l1_loss", start=0)
        F.load_state_dict(snap)
        got.append(step(udh, F, batch(udh, 1)))
        del F
    for g in got:
        assert torch.equal(g["pred"], ref["pred"])
    r_cont = worst_grad_rel_l2(udh, got[0]["grads"], ref["grads"])
    r_fresh = worst_grad_rel_l2(udh, got[0]["grads"], got[1]["grads"])
    print("l1_loss resume: worst per-tensor gradient rel L2 vs continued %.2e, between two resumed runs %.2e" % (r_cont, r_fresh))
    assert r_cont <= GRAD_ENVELOPE and r_fresh <= GRAD_ENVELOPE


def test_resume_through_checkpoints_and_eval(udh, tmp_path):
    """bf16x3: restoring through the TF checkpoint and through a .pt state_dict reproduces the next step bit for bit, and an
    eval_step between two train steps changes nothing."""
    E = make_engine(udh, "bf16x3")
    step(udh, E, batch(udh, 0))
    prefix = str(tmp_path / ("model.ckpt-%d" % E.global_step))
    E.save_tf_checkpoint(prefix)
    torch.save(E.state_dict(), str(tmp_path / "state.pt"))
    ref = step(udh, E, batch(udh, 1))
    F = make_engine(udh, "bf16x3", start=0)
    F.load_tf_checkpoint(prefix)
    assert F.global_step == START + 1
    assert_same(ref, step(udh, F, batch(udh, 1)), "TF checkpoint resume")
    G = make_engine(udh, "bf16x3", start=0)
    G.load_state_dict(torch.load(str(tmp_path / "state.pt")))
    assert_same(ref, step(udh, G, batch(udh, 1)), ".pt resume")
    del F, G
    H = make_engine(udh, "bf16x3")
    step(udh, H, batch(udh, 0))
    H.eval_step(batch(udh, 5))
    got = step(udh, H, batch(udh, 1))
    assert_same(ref, got, "eval between steps", keys=("pred", "metrics", "grads", "params", "m", "v", "mirror"))


def test_two_engines_interleaved(udh):
    """A bf16x3 B = 128 engine and an fp32 B = 4 engine alternating step by step (they share the slab scratch and the
    library's global knobs): the bf16x3 engine equals itself run alone bit for bit over three steps, the fp32 engine's first
    step equals its lone run to GRAD_ENVELOPE."""
    small = {k: v[:4].contiguous() for k, v in batch(udh, 7).items()}
    flat = udh.params.init_flat_large(3)

    def run(interleave):
        big = make_engine(udh, "bf16x3", flat=flat)
        little = make_engine(udh, "fp32", batch_size=4, flat=flat)
        rb, rl = [], []
        for k in range(3):
            rb.append(step(udh, big, batch(udh, k)))
            if interleave:
                rl.append(step(udh, little, small))
        if not interleave:
            for k in range(3):
                rl.append(step(udh, little, small))
        return rb, rl

    alone = run(False)
    both = run(True)
    for a, b in zip(alone[0], both[0]):
        assert_same(a, b, "interleaved bf16x3")
    # the fp32 engine's backward accumulates with atomics, so only its first step starts from identical state
    a, b = alone[1][0], both[1][0]
    assert torch.equal(a["pred"], b["pred"]) and worst_grad_rel_l2(udh, a["grads"], b["grads"]) <= GRAD_ENVELOPE


# ------------------------------------------------------------------------------------------------ 5. scheduling and host API
@pytest.mark.parametrize("numeric", ["bf16x3", "bf16"])
def test_overlapped_update_is_bit_identical(udh, numeric, monkeypatch):
    """UDH_OVERLAP_UPDATE=1 runs the head slice's Adam on a second stream under the conv backward: 4 steps bit-identical
    to the default engine's; afterwards a plain Adam call still matches float64."""
    ref = make_engine(udh, numeric)
    rr = [ref.train_step(batch(udh, k)) and (ref.params.clone(), ref.adam_m.clone(), ref.adam_v.clone(), mirror_of(ref))
          for k in range(4)]
    del ref
    monkeypatch.setenv("UDH_OVERLAP_UPDATE", "1")
    e = make_engine(udh, numeric)
    assert e._overlap_update
    for k in range(4):
        out = e.train_step(batch(udh, k))
        got = (e.params.clone(), e.adam_m.clone(), e.adam_v.clone(), mirror_of(e))
        for name, a, b in zip(("params", "m", "v", "mirror"), rr[k], got):
            assert torch.equal(a, b), "%s overlap step %d: %s" % (numeric, k, name)
    assert (e.grads[:e._mirror[1]] == 0).all() and (e.grads[e._mirror[1] + e._mirror[2]:] == 0).all()
    del e
    rng = np.random.default_rng(3)
    p, g, m, v = (torch.from_numpy(x) for x in Q.adam_inputs(rng, 4132))
    out = run_adam(udh, p, g, m, v, np.float32(1e-3), 1.0, None, 1)
    check_run("adam.after_overlap", out, p, g, m, v, np.float32(1e-3), 1.0, None, 1)


def test_host_stepper_ring_equals_train_step(udh):
    """Six distinct pinned batches through HostStepper.step (ring depth 2) equal train_step on device copies bit for bit, and
    every call returns the previous step's results; the same for step_u8 against prep_u8 + train_step."""
    T = udh.trainer
    names = ("h_loss", "bounded_h_loss", "num_fail", "ace")
    bs = [batch(udh, k, rgb=True) for k in range(6)]
    host = []
    for b in bs:
        hb = {k: b[k].cpu().pin_memory() for k in ("I1_aug", "I2_aug", "I_aug", "pts1", "gt")}
        hb["patch_origin"] = b["patch_indices"].cpu().to(torch.int32).pin_memory()
        host.append(hb)
    ref = make_engine(udh, "bf16x3")
    want = []
    for b in bs:
        out = ref.train_step(b)
        want.append(ref.losses_dict(out))
    ref_state = (ref.params.clone(), ref.adam_m.clone())
    del ref
    e = make_engine(udh, "bf16x3")
    hs = T.HostStepper(e)
    got = [hs.step(hb) for hb in host] + [hs.flush()]
    assert got[0] is None
    for k in range(6):
        for n in names:
            assert got[k + 1][n] == want[k][n], (k, n)
    assert torch.equal(e.params, ref_state[0]) and torch.equal(e.adam_m, ref_state[1])
    del e, hs
    # step_u8: the device prep of the u8 images, then the step
    ref = make_engine(udh, "bf16x3")
    want = []
    for b in bs:
        d = udh.synthetic.prep_u8(b["I_u8"], b["I_prime_u8"], b["pts1"], None)
        d["gt"] = b["gt"]
        want.append(ref.losses_dict(ref.train_step(d)))
    ref_p = ref.params.clone()
    del ref
    e = make_engine(udh, "bf16x3")
    hs = T.HostStepper(e)
    got = [hs.step_u8(T.pin_batch_u8(b["I_u8"], b["I_prime_u8"], b["pts1"], b["gt"])) for b in bs] + [hs.flush()]
    assert got[0] is None
    for k in range(6):
        for n in names:
            assert got[k + 1][n] == want[k][n], ("u8", k, n)
    assert torch.equal(e.params, ref_p)
