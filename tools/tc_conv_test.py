"""Layer-by-layer check of the wgmma conv kernel against torch conv2d on bf16-rounded inputs (GPU)."""
import ctypes, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
print("importing torch", flush=True)
import torch
import torch.nn.functional as F
from unsuperviseddeephomographyral2018_b200 import _lib
lib = _lib.lib
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None

def run(B, H, cin, cout, relu, dgrad, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    kin, kout = (cout, cin) if dgrad else (cin, cout)
    x = torch.randn(B, H, H, kin, device="cuda", generator=g).bfloat16().float().contiguous()
    w = (torch.randn(3, 3, cin, cout, device="cuda", generator=g) * 0.05).bfloat16().float().contiguous()
    bias = torch.randn(kout, device="cuda", generator=g).contiguous() if not dgrad else None
    out = torch.full((B, H, H, kout), float("nan"), device="cuda")
    nb = lib.udh_debug_tc_conv_scratch_bytes(B, H, H, cin, cout)
    scratch = torch.empty(nb, device="cuda", dtype=torch.uint8)
    rc = lib.udh_debug_tc_conv(P(x), P(w), P(bias), P(out), P(scratch), B, H, H, cin, cout, relu, dgrad, None)
    assert rc == 0, lib.udh_last_error()
    torch.cuda.synchronize()
    if dgrad:
        wk = torch.flip(w, dims=(0, 1)).permute(2, 3, 0, 1)          # out-ch = ci, in-ch = co, mirrored taps
    else:
        wk = w.permute(3, 2, 0, 1)
    ref = F.conv2d(x.permute(0, 3, 1, 2), wk.contiguous(), bias, padding=1)
    if relu:
        ref = F.relu(ref)
    ref = ref.permute(0, 2, 3, 1)
    err = (out - ref).abs().max().item()
    nan = torch.isnan(out).float().mean().item()
    print("B=%d H=%3d %3d->%3d relu=%d dgrad=%d  max|err|=%.3e  (ref max %.2f, nan frac %.4f)" % (B, H, cin, cout, relu, dgrad, err, ref.abs().max().item(), nan), flush=True)
    return err

cases = [(2, 128, 64, 64, 1, 0), (3, 64, 64, 64, 1, 0), (2, 32, 64, 128, 1, 0), (2, 32, 128, 128, 0, 0), (5, 16, 128, 128, 1, 0),
         (2, 32, 64, 128, 0, 1), (2, 128, 64, 64, 0, 1), (3, 16, 128, 128, 0, 1)]
for c in cases:
    try:
        run(*c)
    except Exception as e:
        print("case", c, "FAILED:", repr(e)[:300], flush=True)
        break

def run_wgrad(B, H, cin, cout, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, H, H, cin, device="cuda", generator=g).bfloat16().float().contiguous()
    go = (torch.randn(B, H, H, cout, device="cuda", generator=g) * 0.1).bfloat16().float().contiguous()
    dW = torch.zeros(3, 3, cin, cout, device="cuda"); db = torch.zeros(cout, device="cuda")
    nb = lib.udh_debug_tc_conv_scratch_bytes(B, H, H, cin, cout)
    scratch = torch.empty(nb, device="cuda", dtype=torch.uint8)
    rc = lib.udh_debug_tc_wgrad(P(x), P(go), P(dW), P(db), P(scratch), B, H, H, cin, cout, None)
    assert rc == 0, lib.udh_last_error()
    torch.cuda.synchronize()
    ref = torch.nn.grad.conv2d_weight(x.permute(0, 3, 1, 2), (cout, cin, 3, 3), go.permute(0, 3, 1, 2), padding=1).permute(2, 3, 1, 0)
    refb = go.sum(dim=(0, 1, 2))
    e = (dW - ref).abs().max().item(); eb = (db - refb).abs().max().item()
    print("wgrad B=%d H=%3d %3d->%3d  max|err dW|=%.3e (ref max %.2f)  max|err db|=%.3e (ref max %.2f)" % (B, H, cin, cout, e, ref.abs().max().item(), eb, refb.abs().max().item()), flush=True)

for c in [(2, 128, 64, 64), (3, 64, 64, 64), (2, 32, 64, 128), (2, 32, 128, 128), (5, 16, 128, 128)]:
    try:
        run_wgrad(*c)
    except Exception as e:
        print("wgrad case", c, "FAILED:", repr(e)[:300], flush=True)
        break
