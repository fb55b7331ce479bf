"""Exposure-compensation timing, in one run on the GPU, on the synthetic camera sweeps of tools/mosaic_time.py (32 x
1080x1920 and 16 x 3000x4000 RGB frames, about 60 % overlap between neighbours, placed with their true homographies):
  * udh_mosaic_exposure_stats_u8 alone (one feed, frame table and pair list built once, CUDA events over repeated
    launches), without and with the norm sums (channels and gain mode);
  * the whole compensation, ops.mosaic_exposure_gains in both modes with 1 feed (statistics, read-back, the host's
    system and cv2.solve), wall time per call after a warm-up;
  * cv2.detail_GainCompensator / ChannelsCompensator's feed on the same ROI warps and masks (the oracle, CPU) with
    cv2.setNumThreads(1) and (16); the ROI warps are made once and not timed;
  * the blends with and without gains: udh_mosaic_blend_u8 (feather 64) and udh_mosaic_multiband_u8 (5 bands),
    CUDA events over repeated launches (mosaic_time.blend_time).
Prints one JSON line with the card name, power limit and maximum SM clock read in the same run.

    python tools/exposure_time.py
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import exposure as EX  # noqa: E402
from tools import jpeg_time, mosaic_time  # noqa: E402
from tools.mosaic_time import _p, _stream, events_ms  # noqa: E402
from unsuperviseddeephomographyral2018_b200 import _lib, ops  # noqa: E402


def stats_time(dev, M, canvas, reps=10):
    st = ops._ExposureStats(dev, M, canvas[0], canvas[1])
    out = {"pairs": len(st.j)}
    for norms in (0, 1):
        call = lambda: _lib.check(_lib.lib.udh_mosaic_exposure_stats_u8(
            st.ptrs, st.sz.ctypes.data, _p(st.M_d), st.rr.ctypes.data, st.m, _p(st.ptr_d), _p(st.pj_d), len(st.j), None, 0, norms,
            canvas[0], canvas[1], _p(st.out), _p(st.ws), st.nb, _stream()), "udh_mosaic_exposure_stats_u8")
        out["stats_ms_" + ("gain" if norms else "channels")] = events_ms(call, reps)
    return out


def gains_time(dev, M, canvas, reps=3):
    out = {}
    for mode in ("gain", "channels"):
        ops.mosaic_exposure_gains(dev, M, canvas[0], canvas[1], mode, 1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            ops.mosaic_exposure_gains(dev, M, canvas[0], canvas[1], mode, 1)
        out["gains_ms_" + mode] = (time.perf_counter() - t0) * 1e3 / reps
    return out


def cv2_time(frames, M, canvas):
    import cv2
    take, imgs, masks, tls = EX.fed(frames, M, canvas[0], canvas[1])
    out = {}
    for t in (1, 16):
        cv2.setNumThreads(t)
        for mode in ("gain", "channels"):
            t0 = time.perf_counter()
            EX.cv2_gains(imgs, masks, tls, mode, 1)
            out["cv2_feed_ms_%s_threads_%d" % (mode, t)] = (time.perf_counter() - t0) * 1e3
    cv2.setNumThreads(-1)
    return out


def main():
    torch.cuda.set_device(0)
    out = {"gpu": torch.cuda.get_device_name(0), "card": jpeg_time.card()}
    for n, h, w in ((32, 1080, 1920), (16, 3000, 4000)):
        frames, M, canvas = mosaic_time.placed_sweep(n, h, w)
        dev = [torch.from_numpy(f).cuda() for f in frames]
        r = {"canvas": list(canvas)}
        r.update(stats_time(dev, M, canvas))
        r.update(gains_time(dev, M, canvas))
        g = torch.from_numpy(np.random.default_rng(0).uniform(0.8, 1.25, (len(dev), 3))).cuda()
        r.update(mosaic_time.blend_time(dev, M, canvas, gains=g))
        print(json.dumps(r), flush=True)
        r.update(cv2_time(frames, M, canvas))
        out["sweep_%dx%dx%d" % (n, h, w)] = r
        print(json.dumps(r), flush=True)
        del frames, dev
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
