"""CUDA-event time per launch of udh_prep_inputs_u8_ex at the train step's shape (B = 128, 240 x 320, 128 x 128 patches,
gray warp source and both patch pairs, as HostStepper calls it), with no augmentation, with every sample augmented, and
with half of them.  Inputs rotate through more than L2 holds.  `--lib` times another build of libudh (compare two builds
by alternating runs of this script in one session)."""
import argparse
import ctypes
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from unsuperviseddeephomographyral2018_b200 import _lib, synthetic  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--lib", default=_lib.LIB_PATH, help="the libudh build to time (default: the package's)")
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--iters", type=int, default=200)
args = ap.parse_args()

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip())
B, Hh, W, P, NB = 128, 240, 320, 128, 6
dev = torch.device("cuda")
p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
lib = _lib.lib if args.lib == _lib.LIB_PATH else ctypes.CDLL(args.lib)
fn = lib.udh_prep_inputs_u8_ex
fn.restype, fn.argtypes = _lib.SIGNATURES["udh_prep_inputs_u8_ex"]

g = torch.Generator(device=dev).manual_seed(3)
I = [torch.randint(0, 256, (B, Hh, W, 3), device=dev, dtype=torch.uint8, generator=g) for _ in range(NB)]
Ip = [torch.randint(0, 256, (B, Hh, W, 3), device=dev, dtype=torch.uint8, generator=g) for _ in range(NB)]
x0 = torch.randint(45, 148, (B,), device=dev, generator=g); y0 = torch.randint(45, 68, (B,), device=dev, generator=g)
pts1 = torch.stack([x0, y0, x0 + P, y0, x0 + P, y0 + P, x0, y0 + P], 1).float().contiguous()
augs = {"none": None,
        "all": synthetic.draw_augmentation(B, 1.0, "train", g, dev),
        "half": synthetic.draw_augmentation(B, 0.5, "train", g, dev)}
gray = torch.empty(B, Hh, W, 1, device=dev)
outs = [torch.empty(B, P, P, 1, device=dev) for _ in range(4)]
org = torch.empty(B, device=dev, dtype=torch.int32)


def launch(fn, aug, i):
    rc = fn(p(I[i % NB]), p(Ip[i % NB]), p(pts1), p(aug), p(gray), None, p(outs[0]), p(outs[1]), p(outs[2]), p(outs[3]), p(org),
            B, Hh, W, P, None)
    assert rc == 0, rc


def timed(fn, aug):
    for i in range(20):
        launch(fn, aug, i)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for i in range(args.iters):
        launch(fn, aug, i)
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / args.iters


sc = lib.udh_synth_scene_u8
sc.restype, sc.argtypes = _lib.SIGNATURES["udh_synth_scene_u8"]
sc_pts, sc_gt = torch.empty(B, 8, device=dev), torch.empty(B, 8, device=dev)


def timed_scene():
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for i in range(5):
        assert sc(p(I[i % NB]), p(sc_pts), p(sc_gt), B, Hh, W, P, 45, i, None) == 0
    torch.cuda.synchronize(); e0.record()
    for i in range(args.iters // 4):
        sc(p(I[i % NB]), p(sc_pts), p(sc_gt), B, Hh, W, P, 45, i, None)
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (args.iters // 4)


res = {k: [] for k in augs}
scene = []
for r in range(args.rounds):
    for k, aug in augs.items():
        res[k].append(timed(fn, aug))
    scene.append(timed_scene())
print("%s udh_synth_scene_u8 B=%d: median %.1f us/launch" % (os.path.basename(args.lib), B, np.median(scene)))
byts = B * Hh * W * (3 + 3 + 4) + 4 * B * P * P * 4
for k, v in res.items():
    print("%s aug %-4s: median %.1f us/launch (rounds %s), %.0f GB/s algorithmic"
          % (os.path.basename(args.lib), k, np.median(v), " ".join("%.1f" % x for x in v), byts / np.median(v) / 1e3))
