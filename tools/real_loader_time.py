#!/usr/bin/env python
"""Real-data loader throughput, host vs device, and the real-data direct-method harness's seconds per batch.

Writes a generated on-disk real-data set (half the pairs at the full size 240 x 320, half at the network size 142 x 190,
baseline JPEGs as cv2.imwrite writes them) to a temporary directory, then times
  host    Dataloader._disk_batch_extended_host: cv2 decode + uint8 resize, NumPy augment, cv2 fp32 resize per sample;
  device  Dataloader.next_batch: device JPEG decode (+ uint8 upscale of the network-size files), udh_real_prep;
  ecc     homography_conventional_real.run_batch --method direct on one batch (GPU time, CUDA events).
Every timed window ends in a device synchronise.  Prints one JSON line with the card's name, power limit and clocks.

    python tools/real_loader_time.py [--batch 128] [--pairs 512] [--batches 8] [--iters 100]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [s.strip() for s in out.splitlines()[0].split(",")]))
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def write_set(root, n, seed=0):
    import cv2
    from oracle import jpeg as J
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "I")); os.makedirs(os.path.join(root, "I_prime"))
    names, pts1, gt = [], [], []
    for i in range(n):
        name = "%06d.jpg" % i
        h, w = (240, 320) if i % 2 == 0 else (142, 190)
        for sub in ("I", "I_prime"):
            cv2.imwrite(os.path.join(root, sub, name), J.textured(rng, h, w, 3)[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, 95])
        names.append("%s %s" % (name, name))
        x0, y0 = rng.integers(24, 190 - 24 - 128 + 1), rng.integers(4, 142 - 4 - 128 + 1)
        pts1.append([x0, y0, x0 + 128, y0, x0 + 128, y0 + 128, x0, y0 + 128])
        c1 = rng.uniform(80, 560, 8)
        gt.append(np.concatenate([c1, c1 + rng.normal(0, 6, 8)]))
    with open(os.path.join(root, "test_real.txt"), "w") as f:
        f.write("\n".join(names) + "\n")
    np.savetxt(os.path.join(root, "test_pts1.txt"), np.array(pts1, np.float64))
    np.savetxt(os.path.join(root, "test_gt.txt"), np.array(gt, np.float64))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--pairs", type=int, default=512)
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--iters", type=int, default=100)
    a = ap.parse_args()
    import torch
    import homography_conventional_real as M
    from unsuperviseddeephomographyral2018_b200 import _lib
    _lib.require_device()
    res = dict(gpu=gpu_info(), batch=a.batch, pairs=a.pairs, batches=a.batches, ecc_iterations=a.iters)
    with tempfile.TemporaryDirectory() as root:
        write_set(root, a.pairs)
        args = M.resolve_paths(M.build_parser().parse_args(["--method", "direct", "--data_path", root + "/", "--do_augment", "0.5",
                                                            "--num_iterations", str(a.iters), "--log_dir", os.path.join(root, "l"),
                                                            "--results_dir", os.path.join(root, "r")]))
        for arm in ("host", "device"):
            loader = M.make_loader(args, a.batch)
            get = loader._disk_batch_extended_host if arm == "host" else loader.next_batch
            b = get()                                                   # warm-up (device: first decode group, module load)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.batches):
                b = get()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            res[arm + "_batches_per_s"] = a.batches / dt
            res[arm + "_pairs_per_s"] = a.batches * a.batch / dt
        M.run_batch("direct", b, a.iters)                              # warm-up
        secs = [M.run_batch("direct", b, a.iters)[2] for _ in range(3)]
        res["ecc_s_per_batch"] = float(np.median(secs))
        res["ecc_s_per_pair_batched"] = res["ecc_s_per_batch"] / a.batch
    print(json.dumps(res))


if __name__ == "__main__":
    main()
