"""Worker of tests/test_gpu_pdl.py: runs the train step in every numeric mode, loss, batch size and entry point and saves
what each step produced, so that a run with programmatic dependent launch (the default) can be compared with one under
UDH_PDL=0 (plain launches).  pdl_enabled() reads the environment once per process, so each arm is a process of its own.

Usage: python tests/_pdl_worker.py OUT.pt

Large tensors (parameters, gradients, Adam's m and v, fc1's weight mirror) are saved as a fingerprint of all their bits
plus a fixed sample for the relative-L2 comparison: every tensor whole, except fc1's 33.5 M weights, of which every 31st."""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from unsuperviseddeephomographyral2018_b200 import _lib, engine as en, ops, params as P, synthetic, trainer  # noqa: E402

MODES = ("fp32", "bf16x3", "bf16")
LOSSES = ("h_loss", "l1_loss")
BATCHES = (1, 70, 128)
STEPS = 3
START = 3567                    # global_step of the first step (bench.py's lr schedule crosses a boundary at 3570)
LR, MIN_LR = 5e-4, 0.9e-4
SAMPLE_ABOVE, STRIDE = 1 << 20, 31


def deterministic(numeric, loss):
    """fp32's backward and l1_loss's photometric sums accumulate with float atomics: two runs of those drift apart."""
    return numeric != "fp32" and loss == "h_loss"


_W = {}


def fingerprint(t):
    """Two 64-bit sums over the raw bits of t (plain, and position-weighted): equal for equal tensors, and a changed,
    added or moved element changes them."""
    bits = t.detach().contiguous().view(-1)
    bits = bits.view(torch.int32) if bits.element_size() == 4 else bits.view(torch.int16)
    bits = bits.to(torch.int64)
    n = bits.numel()
    if _W.get("n", 0) < n:
        _W["w"] = (torch.arange(n, device=t.device, dtype=torch.int64) * 2654435761) % 2147483647 + 1
        _W["n"] = n
    return torch.stack([bits.sum(), (bits * _W["w"][:n]).sum()]).cpu()


def sample(flat, specs):
    parts = []
    for s in specs.values():
        x = flat[s.offset:s.offset + s.size]
        parts.append((x[::STRIDE] if s.size > SAMPLE_ABOVE else x).float().cpu())
    return parts


def big(flat, specs):
    return dict(fp=fingerprint(flat), sample=sample(flat, specs))


def mirror(e):
    if e._mirror is None:
        return None
    mp, mb, mc, _ = e._mirror
    off = mp - e.ws.data_ptr()
    limbs = 2 if e.numeric_name == "bf16x3" else 1
    return fingerprint(e.ws[off:off + 2 * limbs * mc].view(torch.int16))


def small(out):
    d = dict(pred=out["pred_h4p"].cpu().clone(), photo=out["photo_losses"].cpu().clone())
    if "h4p_metrics" in out:
        d["metrics"] = out["h4p_metrics"].cpu().clone()
    return d


def state(e, specs):
    return dict(params=big(e.params, specs), m=big(e.adam_m, specs), v=big(e.adam_v, specs), mirror=mirror(e))


def batches(B):
    out = []
    for k in range(STEPS + 1):
        b = synthetic.make_batch_fast(B, seed=4000 + 17 * B + k, want_rgb=True)
        b = {kk: v for kk, v in dict(b, I_aug=b["I_aug_rgb"]).items() if isinstance(v, torch.Tensor)}
        out.append(b)
    return out


def host(b):
    hb = {k: b[k].cpu().pin_memory() for k in ("I1_aug", "I2_aug", "I_aug", "pts1", "gt")}
    hb["patch_origin"] = b["patch_indices"].cpu().to(torch.int32).pin_memory()
    return hb


def run_config(numeric, loss, B, init, specs, res):
    det = deterministic(numeric, loss)
    bs = batches(B)
    res[("inputs", numeric, loss, B)] = [fingerprint(b[k]) for b in bs for k in ("I1_aug", "I2_aug", "I_aug", "pts1", "gt")]
    e = en.HomographyEngine(B, seed=None, numeric=numeric, loss_type=loss, lr=LR, min_lr=MIN_LR)
    e.dropout_seed = 99

    def reset(k):
        # atomics configurations: every step starts from the same state in both runs; deterministic ones chain their steps
        if k == 0 or not det:
            e.load_flat(init)
            e.adam_m.zero_(); e.adam_v.zero_(); e.grads.zero_()
        e.global_step = START + k

    paths = ["fwdbwd", "train_step", "host"] + (["prof"] if B == 128 else [])
    for path in paths:
        hs = trainer.HostStepper(e) if path == "host" else None
        for k in range(STEPS):
            reset(k)
            key = (path, numeric, loss, B, k)
            if path == "fwdbwd":
                a = e._fill_args(bs[k], True)
                e._apply_sm_policy()
                _lib.check(_lib.lib.udh_step_forward_backward(ctypes.byref(a), _lib.STEP_ALL, ops._stream()), "udh_step_forward_backward")
                r = small(e._step_out(bs[k]))
                r["grads"] = big(e.grads, specs)
                e.update()
            elif path in ("train_step", "prof"):
                if path == "prof":
                    _lib.lib.udh_prof_enable(1)
                r = small(e.train_step(bs[k]))
                if path == "prof":
                    torch.cuda.synchronize()
                    _lib.lib.udh_prof_enable(0)
            else:
                hs.step(host(bs[k]))
                r = dict(results=torch.tensor(list(hs.flush().values()), dtype=torch.float64))
            r.update(state(e, specs))
            res[key] = r
        # an eval step after the steps (from the initial state where runs drift)
        if not det:
            reset(0)
        if path == "host":
            hs.step(host(bs[STEPS]), train=False)
            res[(path + ".eval", numeric, loss, B)] = dict(results=torch.tensor(list(hs.flush().values()), dtype=torch.float64))
        else:
            res[(path + ".eval", numeric, loss, B)] = small(e.eval_step(bs[STEPS]))
        del hs
    del e
    torch.cuda.empty_cache()


def main():
    out_path = sys.argv[1]
    _lib.require_device()
    torch.cuda.set_device(0)
    specs = P.param_specs()
    init = P.init_flat_large(3)
    res = {}
    for numeric in MODES:
        for loss in LOSSES:
            for B in BATCHES:
                run_config(numeric, loss, B, init, specs, res)
    torch.cuda.synchronize()
    torch.save(dict(pdl=os.environ.get("UDH_PDL", ""), results=res), out_path)


if __name__ == "__main__":
    main()
