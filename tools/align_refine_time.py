"""Refinement timing (HomographyEstimator.refine and udh_ecc_homography_split), in one run on the GPU:
  * refine time per pair with the default levels and iterations: 1 and 16 pairs of 3000x4000 (12 MP), 128 pairs of
    240x320 and of 1080x1920 (synthetic textured pairs, starting corners 6 px off in the 240x320 frame);
  * the same schedule through cv2 (oracle/ecc_refine.py) with cv2.setNumThreads(1) and (16), on a few of those pairs;
  * the split kernel against the one-CTA kernel on the conventional harness's ECC workload: 128 pairs of 240x320,
    100 iterations (eps < 0: no early stop), the same planes;
  * the launch overhead per iteration (every pair already finished: the kernels' CTAs exit at once);
  * the split kernel's achieved bytes/s on one 12 MP level (16 B of blurred planes read per pixel and iteration: both
    planes in each of the two passes) against the H100 SXM's 3.35 TB/s.
Prints one JSON line with the card name and power limit read in the same run.

    python tools/align_refine_time.py
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

import _refine_pairs as P  # noqa: E402
from oracle import ecc_refine as R  # noqa: E402
from tools import jpeg_time  # noqa: E402
from unsuperviseddeephomographyral2018_b200 import align, ops  # noqa: E402

HBM_TBS = 3.35


def pairs(h, w, n, distinct):
    base = [P.pair(h, w, 100 + s, 6.0) for s in range(distinct)]
    return [base[k % distinct] for k in range(n)]


def device_refine(est, ps, reps=2):
    I1 = [torch.from_numpy(p[0]).cuda() for p in ps]
    I2 = [torch.from_numpy(p[1]).cuda() for p in ps]
    H0 = np.stack([p[3] for p in ps])
    est.refine(I1[:1], I2[:1], H0[:1])                                  # warm-up
    best, wall = None, None
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        H, rho, st, lv = est.refine(I1, I2, H0)
        w = time.perf_counter() - t
        ms = est.last_ms["refine"]
        best = ms if best is None else min(best, ms)
        wall = w if wall is None else min(wall, w)
    err = max(P.corner_error(H[k], ps[k][2], *ps[k][0].shape[:2]) for k in range(len(ps)))
    return {"pairs": len(ps), "ms_per_pair": best / len(ps), "wall_ms_per_pair": 1e3 * wall / len(ps),
            "levels": len(align.refine_level_sizes(*ps[0][1].shape[:2])), "failed": int((st != 0).sum()),
            "worst_corner_error_px": err}


def host_refine(ps, threads):
    cv2.setNumThreads(threads)
    t = time.perf_counter()
    for p in ps:
        R.refine(p[0], p[1], p[3])
    return {"pairs": len(ps), "threads": threads, "ms_per_pair": 1e3 * (time.perf_counter() - t) / len(ps)}


def timed(fn, reps=3):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    fn()
    best = None
    for _ in range(reps):
        ev[0].record()
        out = fn()
        ev[1].record()
        ev[1].synchronize()
        ms = ev[0].elapsed_time(ev[1])
        best = ms if best is None else min(best, ms)
    return best, out


def harness_workload():
    ps = pairs(240, 320, 128, 16)
    T = torch.from_numpy(np.stack([cv2.cvtColor(p[1], cv2.COLOR_RGB2GRAY) for p in ps])).cuda()
    I = torch.from_numpy(np.stack([cv2.cvtColor(p[0], cv2.COLOR_RGB2GRAY) for p in ps])).cuda()
    W0 = torch.from_numpy(np.stack([align.to_level(p[3][None], (240, 320), (240, 320), (240, 320))[0] for p in ps])).cuda()
    out = {}
    for name, fn in (("one_cta", ops.find_homography_ecc), ("split", ops.find_homography_ecc_split)):
        ms, (W, rho, it, st) = timed(lambda: fn(T, I, W0, 100, -1.0))
        out[name] = {"ms": ms, "mean_iterations": float(it.float().mean()), "statuses": np.bincount(st.cpu().numpy(), minlength=3).tolist()}
    a = ops.find_homography_ecc(T, I, W0, 100, -1.0)
    b = ops.find_homography_ecc_split(T, I, W0, 100, -1.0)
    same_it = bool(torch.equal(a[2], b[2]) and torch.equal(a[3], b[3]))
    out["iterations_and_statuses_equal"] = same_it
    # launch overhead: eps = 2 finishes every pair before iteration 1, so each iteration is three launches of exiting CTAs
    ms, _ = timed(lambda: ops.find_homography_ecc_split(T, I, W0, 100, 2.0))
    ms0, _ = timed(lambda: ops.find_homography_ecc_split(T, I, W0, 0, 2.0))
    out["split_launch_overhead_us_per_iteration"] = 1e3 * (ms - ms0) / 100
    return out


def bandwidth_12mp(iters=20):
    p = P.pair(3000, 4000, 7, 2.0)
    T = torch.from_numpy(cv2.cvtColor(p[1], cv2.COLOR_RGB2GRAY)[None]).cuda()
    I = torch.from_numpy(cv2.cvtColor(p[0], cv2.COLOR_RGB2GRAY)[None]).cuda()
    W0 = torch.from_numpy(align.to_level(p[3][None], (3000, 4000), (3000, 4000), (3000, 4000))).cuda()
    ms, (W, rho, it, st) = timed(lambda: ops.find_homography_ecc_split(T, I, W0, iters, -1.0))
    ms0, _ = timed(lambda: ops.find_homography_ecc_split(T, I, W0, 0, -1.0))          # init + blur
    n = int(it[0])
    per_it = (ms - ms0) / max(n, 1)
    gbs = 16.0 * 3000 * 4000 / (per_it * 1e-3) / 1e9
    return {"iterations": n, "ms_per_iteration": per_it, "blur_and_init_ms": ms0, "achieved_GBs": gbs, "fraction_of_3.35TBs": gbs / (HBM_TBS * 1e3)}


def main():
    torch.cuda.set_device(0)
    out = {"gpu": torch.cuda.get_device_name(0), "card": jpeg_time.card(), "levels": "default (None)", "iters": align.REFINE_ITERS,
           "eps": align.REFINE_EPS}
    est = align.HomographyEstimator(batch_size=2)
    out["harness_128x240x320_100it"] = harness_workload()
    out["split_12mp_level"] = bandwidth_12mp()
    big = pairs(3000, 4000, 16, 4)
    out["device"] = {"12MP_x1": device_refine(est, big[:1]), "12MP_x16": device_refine(est, big, reps=1),
                     "240x320_x128": device_refine(est, pairs(240, 320, 128, 16)),
                     "1080x1920_x128": device_refine(est, pairs(1080, 1920, 128, 8), reps=1)}
    out["cv2"] = {"12MP": [host_refine(big[:1], t) for t in (1, 16)],
                  "240x320": [host_refine(pairs(240, 320, 16, 16), t) for t in (1, 16)],
                  "1080x1920": [host_refine(pairs(1080, 1920, 4, 4), t) for t in (1, 16)]}
    out["card_after"] = jpeg_time.card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
