"""Seam-finding timing, in one run on the GPU, on the synthetic camera sweeps of tools/mosaic_time.py (32 x 1080x1920 and
16 x 3000x4000 RGB frames, about 60 % overlap between neighbours, placed with their true homographies):
  * udh_mosaic_seam_masks_u8 (validity, every intersecting pair's column and row pass, blend masks), CUDA events over
    repeated calls with the frame table and pair list built once; its launch count (udh_launch_count), the pairs, and
    the seam stage alone with the validity and blend-mask launches subtracted (one call without pairs);
  * the blends with and without blend masks: udh_mosaic_blend_u8 (feather 64) and udh_mosaic_multiband_u8 (5 bands),
    CUDA events over repeated launches (mosaic_time.blend_time);
  * cv2.detail's Voronoi seam finder on the same validity masks (the oracle, CPU) with cv2.setNumThreads(1) and (16);
    the masks are made once and not timed.
With --finder voronoi gc_color both finders are timed in the same run; gc_color's numbers go under "gc_color":
  * udh_mosaic_seam_gc_masks_u8 on every pair, one call timed by CUDA events (seconds per sweep; its launches depend on
    how fast each pair's flow settles), and on the pair with the smallest window alone;
  * cv2's GraphCutSeamFinder(COST_COLOR) (oracle/seam_gc.cv2_seams, CPU, its default threads) on that one pair: it
    needs minutes for a whole sweep's windows at these sizes.
With --seam_megapix X the finders also run at cv2's seam scale a = min(1, sqrt(X 1e6 / frame area)), beside the
full-resolution ones, under "scaled_<finder>": the stages apart (the INTER_LINEAR_EXACT downscale of every frame, the
finder on the seam-scale frames, the upscale to graded blend masks), the whole stage as ops.mosaic_seam_masks(scale=a)
runs it with its launch count, the blends fed the graded masks, and cv2's finder on every pair at seam scale (the
graph-cut one on the whole sweep's seam-scale windows).
Prints one JSON line with the card name, power limit and maximum SM clock read in the same run.

    python tools/seam_time.py [--finder voronoi|gc_color ...] [--seam_megapix X]
"""
import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import seam as SM  # noqa: E402
from oracle import seam_gc as GC  # noqa: E402
from oracle import seam_scale as SS  # noqa: E402
from tools import jpeg_time, mosaic_time  # noqa: E402
from tools.mosaic_time import _p, _stream, events_ms  # noqa: E402
from unsuperviseddeephomographyral2018_b200 import _lib, mosaic, ops  # noqa: E402


def seam_time(dev, M, canvas, reps=5, finder="voronoi", only=None):
    """The seam call on every intersecting pair (or only on pair only = (i, j)) and without pairs -> (times, blend masks)."""
    Hc, Wc = canvas
    n = len(dev)
    sizes = [tuple(int(v) for v in t.shape[:2]) for t in dev]
    rois, Mr = mosaic.multiband_rois(M, sizes, Hc, Wc)
    rr = np.ascontiguousarray(rois.astype(np.int32))
    Mr_d = torch.from_numpy(np.ascontiguousarray(Mr.reshape(n, 9))).cuda()
    sz = np.ascontiguousarray(np.array(sizes, np.int32))
    ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t in dev])
    area = ((rr[:, 2] - rr[:, 0]) * (rr[:, 3] - rr[:, 1])).astype(np.int64)
    seam = torch.empty(int(area.sum()), dtype=torch.uint8, device="cuda")
    blend = torch.empty_like(seam)
    gc = finder == "gc_color"
    pairs = ops.roi_pairs(rr, False)
    if only is not None:
        pairs = (np.array([0] * (only[0] + 1) + [1] * (n - only[0]), np.int32), np.array([only[1]], np.int32))
    res = {}
    for label, (ptr, pj) in (("seam", pairs), ("no_pairs", (np.zeros(n + 1, np.int32), np.zeros(1, np.int32)))):
        ws_bytes = _lib.lib.udh_mosaic_seam_gc_workspace_bytes if gc else _lib.lib.udh_mosaic_seam_workspace_bytes
        nb = ws_bytes(rr.ctypes.data, n, ptr.ctypes.data, pj.ctypes.data, Hc, Wc)
        ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
        args = (ptrs, sz.ctypes.data, _p(Mr_d), rr.ctypes.data, n, ptr.ctypes.data, pj.ctypes.data, Hc, Wc, _p(seam), _p(blend))
        if gc:
            call = lambda: _lib.check(_lib.lib.udh_mosaic_seam_gc_masks_u8(*args, None, _p(ws), nb, _stream()), "udh_mosaic_seam_gc_masks_u8")
        else:
            call = lambda: _lib.check(_lib.lib.udh_mosaic_seam_masks_u8(*args, _p(ws), nb, _stream()), "udh_mosaic_seam_masks_u8")
        l0 = _lib.lib.udh_launch_count()
        if gc:                                                     # seconds per call: the timed call is the only one
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            e1.synchronize()
            res[label + "_ms"] = e0.elapsed_time(e1)
        else:
            call()
            torch.cuda.synchronize()
        res[label + "_launches"] = int(_lib.lib.udh_launch_count() - l0)
        if not gc:
            res[label + "_ms"] = events_ms(call, reps)
        if label == "seam":
            res["pairs"] = int(ptr[-1])
            res["workspace_mb"] = nb / 2 ** 20
    res["pair_loop_ms"] = res["seam_ms"] - res["no_pairs_ms"]
    res["pair_loop_us_per_pair"] = 1e3 * res["pair_loop_ms"] / max(res["pairs"], 1)
    return res, [blend[int(a):int(b)] for a, b in zip(np.concatenate([[0], np.cumsum(area)[:-1]]), np.cumsum(area))]


def cv2_time(frames, M, canvas):
    import cv2
    _, _, masks, tls = SM.fed(frames, M, canvas[0], canvas[1])
    out = {}
    for t in (1, 16):
        cv2.setNumThreads(t)
        t0 = time.perf_counter()
        SM.cv2_seams(masks, tls)
        out["cv2_seam_ms_threads_%d" % t] = (time.perf_counter() - t0) * 1e3
    cv2.setNumThreads(-1)
    return out


def gc_time(frames, dev, M, canvas, cv2_pair=True):
    """The graph-cut finder on the whole sweep and on its smallest pair window, and cv2's on that pair."""
    r, _ = seam_time(dev, M, canvas, finder="gc_color")
    print(json.dumps(r), flush=True)
    _, imgs, masks, tls = SM.fed(frames, M, canvas[0], canvas[1])
    i, j, (x0, y0, x1, y1) = min(SM.pairs(tls, [m.shape for m in masks]), key=lambda p: (p[2][2] - p[2][0]) * (p[2][3] - p[2][1]))
    one, _ = seam_time(dev, M, canvas, finder="gc_color", only=(i, j))
    r.update(small_pair=[i, j], small_pair_window=[y1 - y0 + 2 * SM.GAP, x1 - x0 + 2 * SM.GAP], small_pair_ms=one["pair_loop_ms"],
             small_pair_launches=one["seam_launches"] - one["no_pairs_launches"])
    if cv2_pair:
        t0 = time.perf_counter()
        GC.cv2_seams([imgs[i], imgs[j]], [masks[i], masks[j]], [tls[i], tls[j]])
        r["cv2_small_pair_ms"] = (time.perf_counter() - t0) * 1e3
    print(json.dumps(r), flush=True)
    return r


def upscale_time(dev, M, canvas, a, found, seam_canvas, reps=10):
    """udh_mosaic_seam_upscale_u8 alone on the seam-scale seams `found` (ops.mosaic_seam_masks at seam scale) -> ms."""
    Hc, Wc = canvas
    n = len(dev)
    sizes = [tuple(int(v) for v in t.shape[:2]) for t in dev]
    rois, Mr = mosaic.multiband_rois(M, sizes, Hc, Wc)
    rr = np.ascontiguousarray(rois.astype(np.int32))
    srr = np.zeros((n, 4), np.int32)
    sp = (ctypes.c_void_p * n)()
    for q, k in enumerate(found["take"]):
        srr[k] = found["rois"][k]
        sp[k] = found["seam"][q].data_ptr()
    Mr_d = torch.from_numpy(np.ascontiguousarray(Mr.reshape(n, 9))).cuda()
    sz = np.ascontiguousarray(np.array(sizes, np.int32))
    ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t in dev])
    blend = torch.empty(int(((rr[:, 2] - rr[:, 0]) * (rr[:, 3] - rr[:, 1]).astype(np.int64)).sum()), dtype=torch.uint8, device="cuda")
    Hs, Ws = seam_canvas
    nb = _lib.lib.udh_mosaic_seam_upscale_workspace_bytes(rr.ctypes.data, srr.ctypes.data, n, Hs, Ws, a, Hc, Wc)
    ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
    call = lambda: _lib.check(_lib.lib.udh_mosaic_seam_upscale_u8(ptrs, sz.ctypes.data, _p(Mr_d), rr.ctypes.data, sp, srr.ctypes.data, n, Hs,
                                                                  Ws, a, Hc, Wc, _p(blend), _p(ws), nb, _stream()), "udh_mosaic_seam_upscale_u8")
    return events_ms(call, reps)


def scaled_time(frames, dev, M, canvas, megapix, finder, cv2_all=True):
    """The seam stage at cv2's seam scale for megapix: its three stages apart, whole, the blends with its graded masks and
    cv2's finder on every seam-scale pair."""
    Hc, Wc = canvas
    a = mosaic.seam_scale([f.shape[:2] for f in frames], megapix)
    Ms, _, seam_canvas = mosaic.seam_geometry(M, [f.shape[:2] for f in frames], Hc, Wc, a)
    r = {"scale": a, "seam_canvas": list(seam_canvas)}
    gc = finder == "gc_color"
    r["downscale_ms"] = events_ms(lambda: [ops.resize_linear_exact_u8(t, scale=a) for t in dev], 10)
    small = [ops.resize_linear_exact_u8(t, scale=a) for t in dev]
    find = lambda: ops.mosaic_seam_masks(small, Ms, seam_canvas[0], seam_canvas[1], finder)
    stage = lambda: ops.mosaic_seam_masks(dev, M, Hc, Wc, finder, scale=a)
    found = find()
    torch.cuda.synchronize()
    for label, call in (("finder", find), ("stage", stage)):
        if gc:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            e1.synchronize()
            r[label + "_ms"] = e0.elapsed_time(e1)
        else:
            r[label + "_ms"] = events_ms(call, 10)
    r["upscale_ms"] = upscale_time(dev, M, canvas, a, found, seam_canvas)
    l0 = _lib.lib.udh_launch_count()
    got = stage()
    torch.cuda.synchronize()
    r["stage_launches"] = int(_lib.lib.udh_launch_count() - l0)
    r["pairs"] = int(ops.roi_pairs(np.asarray(found["rois"])[found["take"]], False)[0][-1])
    r.update(mosaic_time.blend_time(dev, M, canvas, masks=got["blend"]))
    print(json.dumps(r), flush=True)
    if cv2_all:
        _, imgs, masks, tls = SM.fed([SS.resize_exact(f, fx=a) for f in frames], Ms, seam_canvas[0], seam_canvas[1])
        t0 = time.perf_counter()
        (GC.cv2_seams(imgs, masks, tls) if gc else SM.cv2_seams(masks, tls))
        r["cv2_all_pairs_ms"] = (time.perf_counter() - t0) * 1e3
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--finder", nargs="+", default=["voronoi"], choices=["voronoi", "gc_color"])
    ap.add_argument("--no_cv2", action="store_true", help="skip cv2's timing")
    ap.add_argument("--seam_megapix", type=float, default=-1, help="also time the finders at this seam scale (-1: no)")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    out = {"gpu": torch.cuda.get_device_name(0), "card": jpeg_time.card(), "finder": args.finder}
    for n, h, w in ((32, 1080, 1920), (16, 3000, 4000)):
        frames, M, canvas = mosaic_time.placed_sweep(n, h, w)
        dev = [torch.from_numpy(f).cuda() for f in frames]
        r = {"canvas": list(canvas)}
        if args.seam_megapix > 0:
            for finder in args.finder:
                r["scaled_" + finder] = scaled_time(frames, dev, M, canvas, args.seam_megapix, finder, not args.no_cv2)
                print(json.dumps(r), flush=True)
        if "voronoi" in args.finder:
            s, bm = seam_time(dev, M, canvas)
            r.update(s)
            r.update(mosaic_time.blend_time(dev, M, canvas, masks=bm))
            print(json.dumps(r), flush=True)
            if not args.no_cv2:
                r.update(cv2_time(frames, M, canvas))
            del bm
        if "gc_color" in args.finder:
            r["gc_color"] = gc_time(frames, dev, M, canvas, not args.no_cv2)
        out["sweep_%dx%dx%d" % (n, h, w)] = r
        print(json.dumps(r), flush=True)
        del frames, dev
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
