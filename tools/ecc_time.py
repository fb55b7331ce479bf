"""Direct-method baseline (cv2.findTransformECC, MOTION_HOMOGRAPHY, 8 iterations) on 240x320 gray planes, B = 128:
CUDA-event time per batch of the blur pre-pass + iterations + corner post-processing, and, where cv2 imports, single-thread
cv2 pairs/s on the same planes.  Prints one JSON line.

    python tools/ecc_time.py [--batch 128] [--iters 10]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from unsuperviseddeephomographyral2018_b200 import ops, synthetic  # noqa: E402


def sm_clock_mhz():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=10).stdout.strip().split(",")
        return {"sm_mhz": float(out[0]), "power_limit_w": float(out[1])}
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    B = args.batch
    sb = synthetic.make_batch_fast(B, seed=31)
    g1, g2 = ops.ecc_prep_u8(sb["I_u8"], sb["I_prime_u8"], None)

    def ecc():
        W, _, _, st = ops.find_homography_ecc(g1, g2, None, 8, 1e-10)
        ops.ecc_h4p(W, st, sb["pts1"], sb["gt"], 45.0)
    for _ in range(2):
        ecc()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(args.iters):
        ecc()
    e1.record(); torch.cuda.synchronize()
    clocks = sm_clock_mhz()
    ms = e0.elapsed_time(e1) / args.iters
    out = {"measurement": "direct method (ECC, 8 iterations), B=%d" % B, "pairs_per_s": B / (ms * 1e-3), "ms_per_batch": ms,
           "gpu": torch.cuda.get_device_name(0), "clocks_after": clocks,
           "what": "blur pre-pass + 8 ECC iterations (one CTA per pair) + corner post-processing on 240x320 gray planes"}
    try:
        import cv2
        cv2.setNumThreads(1)
        n = 4
        G1, G2 = g1[:n].cpu().numpy(), g2[:n].cpu().numpy()
        crit = (cv2.TERM_CRITERIA_EPS | cv2.TERM_CRITERIA_COUNT, 8, 1e-10)
        t0 = time.perf_counter()
        for s in range(n):
            try:
                cv2.findTransformECC(G1[s], G2[s], np.eye(3, dtype=np.float32), cv2.MOTION_HOMOGRAPHY, crit, None, 5)
            except cv2.error:
                pass
        out["cpu_cv2"] = {"pairs_per_s": n / (time.perf_counter() - t0), "threads": 1, "cv2": cv2.__version__,
                          "sample": "%d pairs; pairs where cv2 raises stop early, so this is an upper bound" % n}
    except ImportError:
        out["cpu_cv2"] = None
    print(json.dumps(out))


if __name__ == "__main__":
    main()
