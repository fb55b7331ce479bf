"""The programmatic-dependent-launch chain on the device (DESIGN.md section 2, "The PDL chain").

  * Launch order of the pre-wait readers: conv1_1's forward kernels read the conv1_1 weights before their
    griddepcontrol.wait (tests/_pdl_audit.py, PRE_WAIT_ALLOWED).  That is safe only while the kernel launched right before
    them on their stream waits in its first instruction block (so they start only after everything before it has
    completed) and no kernel that writes the parameters runs on another stream in between.  Checked on torch.profiler
    traces of the train step (bf16x3, bf16), eval_step, the inference forward, HostStepper.step_u8, the overlapped update
    and a step under an SM reserve.  The trace also reports how many chained pairs overlapped.
  * PDL off against PDL on: the whole step in every mode, loss and batch size, through udh_step_forward_backward,
    train_step, HostStepper and the profiled step (udh_prof_enable), run once with UDH_PDL=0 and once without, each in a
    process of its own (tests/_pdl_worker.py).  Deterministic configurations must agree bit for bit; where float atomics
    make two runs drift (fp32's backward, l1_loss's photometric sums) every step starts from the same state and pred_h4p
    must agree bit for bit, everything else within rel-L2 1e-4 per tensor (1e-2 in single-pass bf16), the parameters
    after the update within 1e-2 (5e-2)."""
import json
import os
import subprocess
import sys
import time

import pytest
import torch

import _pdl_audit as A

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B = 128


@pytest.fixture(scope="module")
def udh():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from unsuperviseddeephomographyral2018_b200 import _lib, build_ext, engine, params, synthetic, trainer
    _lib.require_device()

    class NS:
        pass
    ns = NS()
    ns.lib, ns.build_ext, ns.engine, ns.params, ns.synthetic, ns.trainer = _lib, build_ext, engine, params, synthetic, trainer
    return ns


@pytest.fixture(scope="module")
def top_waiters(udh):
    """Kernels of the shipped library whose every instantiation waits in its first instruction block."""
    if A.tool("cuobjdump") is None:
        pytest.skip("cuobjdump is not installed")
    top = {}
    for mangled, insns in A.disassemble(udh.build_ext.LIB).items():
        b = A.base_of_mangled(mangled)
        top[b] = top.get(b, True) and A.waits_first(insns)
    return {b for b, v in top.items() if v}


def chained(udh):
    out = set()
    for s in udh.build_ext.sources():
        out |= A.chained_kernels(udh.build_ext.CSRC, os.path.basename(s))
    return out


def trace(fn, path):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    marker = torch.zeros(4, device="cuda")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        # a few torch kernels first: a trace can miss the first kernel after the profiler starts, and a workload's own
        # first kernel (the weight pack) is the one the check needs
        for _ in range(3):
            marker.add_(1)
        fn()
        torch.cuda.synchronize()
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = json.load(f)["traceEvents"]
    return [(e["args"]["stream"], float(e["ts"]), float(e["ts"]) + float(e["dur"]), e["name"])
            for e in ev if e.get("cat") == "kernel"]


def test_pre_wait_readers_follow_a_waiting_launch(udh, top_waiters, tmp_path, monkeypatch):
    assert {"pack_all_weights_kernel", "pack_all_weights_x3_kernel"} <= top_waiters
    T = udh.trainer
    b = udh.synthetic.make_batch_fast(B, seed=77, want_rgb=True)
    db = {k: v for k, v in dict(b, I_aug=b["I_aug_rgb"]).items() if isinstance(v, torch.Tensor)}
    flat = udh.params.init_flat_large(3)

    def engine(numeric):
        e = udh.engine.HomographyEngine(B, seed=None, numeric=numeric, loss_type="h_loss", lr=5e-4, min_lr=0.9e-4)
        e.load_flat(flat)
        return e

    def stepper(e):
        hs = T.HostStepper(e)
        hb = T.pin_batch_u8(b["I_u8"], b["I_prime_u8"], b["pts1"], b["gt"])
        return lambda: (hs.step_u8(hb), hs.step_u8(hb), hs.flush())

    def reserved(e):
        e._sm_policy = dict(e._sm_policy, reserve=20)
        return lambda: e.train_step(db)

    workloads = [
        ("train_step bf16x3", "bf16x3", lambda e: lambda: e.train_step(db)),
        ("train_step bf16", "bf16", lambda e: lambda: e.train_step(db)),
        ("eval_step bf16x3", "bf16x3", lambda e: lambda: e.eval_step(db)),
        ("forward bf16x3", "bf16x3", lambda e: lambda: e.forward(db, train=False)),
        ("HostStepper.step_u8 bf16x3", "bf16x3", stepper),
        ("overlapped update bf16x3", "bf16x3", None),
        ("SM reserve 20 bf16", "bf16", reserved),
    ]
    ch = chained(udh)
    problems = []
    for name, numeric, make in workloads:
        if make is None:                                   # UDH_OVERLAP_UPDATE=1: the head slice's Adam on a second stream
            monkeypatch.setenv("UDH_OVERLAP_UPDATE", "1")
            e = engine(numeric)
            assert e._overlap_update
            monkeypatch.delenv("UDH_OVERLAP_UPDATE")
            fn = lambda: (e.train_step(db), e.train_step(db))
        else:
            e = engine(numeric)
            fn = make(e)
        fn()                                               # warm-up outside the trace
        ks = trace(fn, str(tmp_path / "trace.json"))
        n, p = A.pre_wait_order_problems(ks, top_waiters)
        pairs, overlap = A.overlapping_pairs(ks, ch)
        print("%-28s kernels %4d  pre-wait readers checked %d  chained pairs %4d, overlapping %d" % (name, len(ks), n, pairs, overlap))
        assert n > 0, "%s: no conv1_1 forward in the trace" % name
        # the H100 traces overlap most chained pairs (e.g. 58 of 62 in the train step): the profiler leaves PDL in effect
        assert overlap > 0, "%s: no chained pair overlapped: PDL did not take effect" % name
        problems += ["%s: %s" % (name, x) for x in p]
        del e
        torch.cuda.empty_cache()
    assert not problems, "\n".join(problems)


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / max(b.norm().item(), 1e-30)).item()


def run_worker(out, pdl):
    env = dict(os.environ, UDH_PDL=pdl)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "_pdl_worker.py"), out], cwd=ROOT, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-6000:]
    return torch.load(out, weights_only=False)


def test_pdl_off_matches_pdl_on(udh, tmp_path):
    t0 = time.time()
    on = run_worker(str(tmp_path / "on.pt"), "1")
    t1 = time.time()
    off = run_worker(str(tmp_path / "off.pt"), "0")
    t2 = time.time()
    print("PDL on: %.1f s, PDL off: %.1f s (worker processes)" % (t1 - t0, t2 - t1))
    assert (on["pdl"], off["pdl"]) == ("1", "0")
    on, off = on["results"], off["results"]
    assert set(on) == set(off) and len(on) > 0
    names = list(udh.params.param_specs())
    bad, worst = [], {}
    for key in sorted(on, key=str):
        a, b = on[key], off[key]
        if key[0] == "inputs":
            assert all(torch.equal(x, y) for x, y in zip(a, b)), "%s: the two runs drew different batches" % (key,)
            continue
        numeric, loss = key[1], key[2]
        det = numeric != "fp32" and loss == "h_loss"
        tol = 1e-2 if numeric == "bf16" else 1e-4
        # Adam's first step from zero moments moves each parameter by about alpha_t * sign(g): a gradient element within
        # rounding of zero may flip its parameter's step, so the parameters get a wider bound than their gradients
        tol_params = 5e-2 if numeric == "bf16" else 1e-2
        for field in sorted(a):
            x, y = a[field], b[field]
            if x is None:
                assert y is None
                continue
            if field == "pred" or det:
                if isinstance(x, dict):
                    same = torch.equal(x["fp"], y["fp"]) and all(torch.equal(u, v) for u, v in zip(x["sample"], y["sample"]))
                else:
                    same = torch.equal(x, y)
                if not same:
                    bad.append("%s %s: not bit-identical" % (key, field))
                continue
            if field == "mirror":                                     # the weights' split: compared through the weights
                continue
            pairs = zip(names, x["sample"], y["sample"]) if isinstance(x, dict) else [("", x, y)]
            for n, u, v in pairs:
                r = rel_l2(u, v)
                w = (numeric, field)
                worst[w] = max(worst.get(w, 0.0), r)
                if r > (tol_params if field == "params" else tol):
                    bad.append("%s %s %s: rel L2 %.2e > %.0e" % (key, field, n, r, tol))
    print("worst rel L2, PDL off vs on, where float atomics let runs drift: " +
          "  ".join("%s/%s %.1e" % (k[0], k[1], v) for k, v in sorted(worst.items())))
    assert not bad, "\n".join(bad[:40])
