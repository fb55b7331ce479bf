"""Block exposure compensation timing, in one run on the GPU, on the synthetic camera sweeps of tools/mosaic_time.py (32 x
1080x1920 and 16 x 3000x4000 RGB frames, about 60 % overlap between neighbours), 32 px blocks:
  * the block and cell counts, and the unknowns of the gain-mode system;
  * udh_mosaic_exposure_block_stats_u8 alone (one feed; without and with the norm sums), CUDA events over repeated
    launches;
  * the host's sparse assembly (wall time), udh_exposure_block_solve (CUDA events, with its iteration count) and
    udh_exposure_gain_maps (CUDA events);
  * the whole ops.mosaic_exposure_gain_maps in both modes with 1 feed, wall time per call after a warm-up;
  * the blends with and without gain maps: udh_mosaic_blend_u8 (feather 64) and udh_mosaic_multiband_u8 (5 bands),
    CUDA events over repeated launches (mosaic_time.blend_time).
cv2.detail_BlocksGainCompensator's dense solve cannot run at these sizes, so it is timed (feed, 1 and 16 threads) on a
small sweep, 8 x 270x480, next to ops.mosaic_exposure_gain_maps on the same frames.  Prints one JSON line per sweep and
one with everything, with the card name, power limit and maximum SM clock read in the same run.

    python tools/exposure_blocks_time.py
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
from oracle import exposure_blocks as XB  # noqa: E402
from tools import jpeg_time, mosaic_time  # noqa: E402
from tools.mosaic_time import _p, _stream, events_ms  # noqa: E402
from unsuperviseddeephomographyral2018_b200 import _lib, ops  # noqa: E402

BLOCK = 32


def stats_time(dev, M, canvas, reps=10):
    st = ops._ExposureBlockStats(dev, M, canvas[0], canvas[1], BLOCK)
    c = st.cells
    out = {"frames": st.m, "blocks": st.nblocks, "block_pairs": len(c["a"]), "cells": int(c["nslots"])}
    for norms in (0, 1):
        call = lambda: _lib.check(_lib.lib.udh_mosaic_exposure_block_stats_u8(
            st.ptrs, st.sz.ctypes.data, _p(st.M_d), st.rr.ctypes.data, st.m, st.blocks.ctypes.data, st.boff.ctypes.data, st.nblocks,
            _p(st.ptr_d), _p(st.pj_d), len(c["pair_j"]), _p(st.off_d), _p(st.nx_d), c["nslots"], None, 0, norms, canvas[0], canvas[1],
            _p(st.out), _p(st.ws), st.nb, _stream()), "udh_mosaic_exposure_block_stats_u8")
        out["stats_ms_" + ("gain" if norms else "channels")] = events_ms(call, reps)
    raw = st(None, True)
    count = raw[:, 0].astype(np.int64)
    pos = count > 0
    sa, sb = np.zeros(len(count)), np.zeros(len(count))
    sa[pos], sb[pos] = ops.exposure_norm_sum(*raw[pos, 7:10].T), ops.exposure_norm_sum(*raw[pos, 10:13].T)
    t0 = time.perf_counter()
    keep, ptr, col, val, rhs = ops.exposure_block_system(st.nblocks, c["a"], c["b"], count, sa, sb)
    out["assembly_ms_host"] = (time.perf_counter() - t0) * 1e3
    out.update(unknowns=len(keep), nonzeros=len(val))
    n = len(keep)
    t = [torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in (ptr, col, val, rhs)]
    x = torch.empty(n, device="cuda", dtype=torch.float64)
    info = torch.zeros(2, device="cuda", dtype=torch.int64)
    nb = _lib.lib.udh_exposure_block_solve_workspace_bytes(n)
    ws = torch.empty(nb, device="cuda", dtype=torch.uint8)
    out["solve_ms"] = events_ms(lambda: _lib.check(_lib.lib.udh_exposure_block_solve(
        n, _p(t[0]), _p(t[1]), _p(t[2]), _p(t[3]), ops.EXPOSURE_BLOCK_TOL, ops.EXPOSURE_BLOCK_MAX_ITER, _p(x), _p(info), _p(ws), nb,
        _stream()), "udh_exposure_block_solve"), 5)
    inf = info.cpu().numpy()
    out["solve_iters"], out["solve_rel_residual"] = int(inf[0]), float(inf[1:2].view(np.float64)[0])
    g = torch.ones(st.nblocks, 3, device="cuda", dtype=torch.float64)
    maps = torch.empty(st.nblocks * 3, device="cuda", dtype=torch.float32)
    nb = _lib.lib.udh_exposure_gain_maps_workspace_bytes(st.nblocks, 3)
    ws = torch.empty(nb, device="cuda", dtype=torch.uint8)
    out["filter_ms"] = events_ms(lambda: _lib.check(_lib.lib.udh_exposure_gain_maps(
        _p(g), st.m, st.blocks.ctypes.data, st.boff.ctypes.data, st.nblocks, 3, _p(maps), _p(ws), nb, _stream()),
        "udh_exposure_gain_maps"), 10)
    return out


def maps_time(dev, M, canvas, reps=3):
    out = {}
    for mode in ("gain", "channels"):
        ops.mosaic_exposure_gain_maps(dev, M, canvas[0], canvas[1], mode, 1, BLOCK)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            ops.mosaic_exposure_gain_maps(dev, M, canvas[0], canvas[1], mode, 1, BLOCK)
        out["gain_maps_ms_" + mode] = (time.perf_counter() - t0) * 1e3 / reps
    return out


def cv2_small():
    """cv2's block compensators on 8 x 270x480 frames (about 1000 blocks: its dense LU still runs) and ours on the same."""
    import cv2
    frames, M, canvas = mosaic_time.placed_sweep(8, 270, 480)
    take, imgs, masks, tls = EX.fed(frames, M, canvas[0], canvas[1])
    out = {"small_sweep": "8x270x480", "small_blocks": len(XB.blocks(imgs, masks, tls, BLOCK, BLOCK)[0])}
    for t in (1, 16):
        cv2.setNumThreads(t)
        for mode in ("gain", "channels"):
            t0 = time.perf_counter()
            XB.cv2_maps(imgs, masks, tls, mode, 1, BLOCK)
            out["cv2_blocks_ms_%s_threads_%d" % (mode, t)] = (time.perf_counter() - t0) * 1e3
    cv2.setNumThreads(-1)
    dev = [torch.from_numpy(f).cuda() for f in frames]
    out.update({"small_" + k: v for k, v in maps_time(dev, M, canvas).items()})
    return out


def main():
    torch.cuda.set_device(0)
    out = {"gpu": torch.cuda.get_device_name(0), "card": jpeg_time.card(), "block": BLOCK}
    out.update(cv2_small())
    print(json.dumps(out), flush=True)
    for n, h, w in ((32, 1080, 1920), (16, 3000, 4000)):
        frames, M, canvas = mosaic_time.placed_sweep(n, h, w)
        dev = [torch.from_numpy(f).cuda() for f in frames]
        r = {"canvas": list(canvas)}
        r.update(stats_time(dev, M, canvas))
        r.update(maps_time(dev, M, canvas))
        r.update(mosaic_time.blend_time(dev, M, canvas, gain_maps=ops.mosaic_exposure_gain_maps(dev, M, canvas[0], canvas[1], "channels", 1,
                                                                                                  BLOCK)))
        out["sweep_%dx%dx%d" % (n, h, w)] = r
        print(json.dumps(r), flush=True)
        del frames, dev
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
