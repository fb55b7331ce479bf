"""Sequence-mosaic timing, in one run on the GPU:
  * udh_mosaic_blend_u8 alone (tile lists built once, CUDA events over repeated launches) on synthetic camera sweeps of
    32 x 1080x1920 and 16 x 3000x4000 RGB frames with about 60 % overlap between neighbours, placed with their true
    homographies: ms per mosaic and bytes/s against the H100 SXM's 3.35 TB/s.  Bytes: the canvas write, (C + 1) per pixel,
    plus C source bytes per covered frame-pixel (each frame's mapped area); candidate frame-pixels (tile pixels times
    candidates, ~12 fp64 operations and one fp64 division each) are printed beside them;
  * the host path, oracle/mosaic.py (cv2.warpPerspective per frame + a NumPy int64 blend), with cv2.setNumThreads(1) and
    (16), against the kernel on the same 8 x 1080x1920 sweep (the oracle evaluates every frame at every canvas pixel);
  * mosaic_images.py end to end (device decode, estimate, chain, blend, JPEG encode, files written) with seeded weights on
    8 quality-95 JPEGs of 1080x1920, ms per frame;
  * the multi-band blend (udh_mosaic_multiband_u8) on the same two sweeps at 5 and 8 bands: CUDA-event ms per mosaic, per
    phase through the library's phase timers (base level, pyramids, accumulate, collapse), bytes moved computed from the
    shapes against 3.35 TB/s, and cv2.detail_MultiBandBlender (the oracle, CPU) on the same frames with 1 and 16 threads
    (the ROI warps and the blender timed apart).
Prints one JSON line with the card name and power limit read in the same run.

    python tools/mosaic_time.py [--legs feather,multiband]
"""
import argparse
import ctypes
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import _mosaic_sweep as SW  # noqa: E402
from tools import jpeg_time  # noqa: E402
from unsuperviseddeephomographyral2018_b200 import _lib, mosaic, ops  # noqa: E402

HBM_TBS = 3.35


def placed_sweep(n, h, w, seed=0):
    """Frames (seeded noise: content does not change the kernel's work) on the canvas of their true homographies."""
    A, _ = SW.sweep_cameras(n, h, w, 0.6, seed)
    G, ref = mosaic.chain_to_reference(SW.true_pairs(A))
    M, (Hc, Wc), kept = mosaic.canvas([(h, w)] * n, G, ref)
    assert kept.all()
    rng = np.random.default_rng(seed)
    frames = [rng.integers(0, 256, (h, w, 3), np.uint8) for _ in range(n)]
    return frames, M, (Hc, Wc)


def mapped_area(M, h, w):
    x, y, _ = mosaic._map(M, mosaic.centre_corners(h, w))
    return 0.5 * abs(np.dot(x, np.roll(y, -1)) - np.dot(y, np.roll(x, -1)))


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def events_ms(call, reps):
    call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


VARIANTS = {"gains": "gain", "masks": "masked", "gain_maps": "gainmap"}


def blend_time(dev, M, canvas, reps=10, **variant):
    """Both blends alone, plain and with one optional input: CUDA events over repeated calls of udh_mosaic_blend_u8 (feather
    64) and udh_mosaic_multiband_u8 (5 bands) on the RGB frames dev (CUDA) placed by M (frame -> canvas), every frame's ROI
    meeting the canvas.  variant: gains= (CUDA float64 [n,3]), masks= ([n] CUDA uint8 blend masks on the ROIs) or
    gain_maps= ([n], as ops.mosaic_exposure_gain_maps gives them).  -> feather_ms, feather_<v>_ms, multiband_ms and
    multiband_<v>_ms, <v> the variant's name in VARIANTS."""
    (kind, value), = variant.items()
    Hc, Wc = canvas
    n = len(dev)
    sizes = [tuple(int(v) for v in t.shape[:2]) for t in dev]
    out_img = torch.empty(Hc, Wc, 3, dtype=torch.uint8, device="cuda")
    mask = torch.empty(Hc, Wc, dtype=torch.uint8, device="cuda")
    ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t in dev])
    sz = np.ascontiguousarray(np.array(sizes, np.int32))
    rois, Mr = mosaic.multiband_rois(M, sizes, Hc, Wc)
    rr = np.ascontiguousarray(rois.astype(np.int32))
    g = value if kind == "gains" else None
    gm, _keep = ops._gain_map_table(value, rr, n, torch.device("cuda"), "blend_time") if kind == "gain_maps" else (None, None)
    mp = (ctypes.c_void_p * n)(*[t.data_ptr() for t in value]) if kind == "masks" else None
    rois_arg = None if kind == "gains" else rr.ctypes.data
    ptr, idx = ops.mosaic_tile_lists(M, sizes, Hc, Wc)
    ptr_d, idx_d = torch.from_numpy(ptr).cuda(), torch.from_numpy(idx).cuda()
    M_d = torch.from_numpy(np.ascontiguousarray(M.reshape(n, 9))).cuda()
    nb = _lib.lib.udh_mosaic_workspace_bytes(n)
    ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
    feather = lambda g, gm, mp, r: lambda: _lib.check(_lib.lib.udh_mosaic_blend_u8(
        ptrs, sz.ctypes.data, _p(M_d), _p(g), gm, mp, r, n, 3, _p(ptr_d), _p(idx_d), Hc, Wc, 64, _p(out_img), _p(mask), _p(ws), nb,
        _stream()), "udh_mosaic_blend_u8")
    res = {"feather_ms": events_ms(feather(None, None, None, None), reps)}
    res["feather_%s_ms" % VARIANTS[kind]] = events_ms(feather(g, gm, mp, rois_arg), reps)
    Mr_d = torch.from_numpy(np.ascontiguousarray(Mr.reshape(n, 9))).cuda()
    nb_mb = _lib.lib.udh_mosaic_multiband_workspace_bytes(rr.ctypes.data, n, Hc, Wc, 5)
    ws_mb = torch.empty(nb_mb, dtype=torch.uint8, device="cuda")
    multiband = lambda g, gm, mp: lambda: _lib.check(_lib.lib.udh_mosaic_multiband_u8(
        ptrs, sz.ctypes.data, _p(Mr_d), _p(g), gm, mp, rr.ctypes.data, n, 3, Hc, Wc, 5, _p(out_img), _p(mask), _p(ws_mb), nb_mb,
        _stream()), "udh_mosaic_multiband_u8")
    res["multiband_ms"] = events_ms(multiband(None, None, None), reps)
    res["multiband_%s_ms" % VARIANTS[kind]] = events_ms(multiband(g, gm, mp), reps)
    return res


def kernel_time(frames, M, canvas, feather=64, reps=10):
    Hc, Wc = canvas
    n, (h, w, C) = len(frames), frames[0].shape
    dev = [torch.from_numpy(f).cuda() for f in frames]
    ptr, idx = ops.mosaic_tile_lists(M, [(h, w)] * n, Hc, Wc)
    ptr_d, idx_d = torch.from_numpy(ptr).cuda(), torch.from_numpy(idx).cuda()
    M_d = torch.from_numpy(np.ascontiguousarray(M.reshape(n, 9))).cuda()
    out = torch.empty(Hc, Wc, C, dtype=torch.uint8, device="cuda")
    mask = torch.empty(Hc, Wc, dtype=torch.uint8, device="cuda")
    nb = _lib.lib.udh_mosaic_workspace_bytes(n)
    ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
    ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t in dev])
    sz = np.array([(h, w)] * n, np.int32)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    call = lambda: _lib.check(_lib.lib.udh_mosaic_blend_u8(ptrs, sz.ctypes.data, p(M_d), None, None, None, None, n, C, p(ptr_d), p(idx_d),
                                                           Hc, Wc, feather, p(out), p(mask), p(ws), nb, st), "udh_mosaic_blend_u8")
    call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / reps
    # the same bytes as ops.mosaic_blend_u8 (its own lists) gives: check the direct call's output once
    ref, ref_mask = ops.mosaic_blend_u8(dev, M, Hc, Wc, feather)
    assert torch.equal(ref, out) and torch.equal(ref_mask, mask)
    covered = sum(mapped_area(M[k], h, w) for k in range(n))
    nbytes = (C + 1) * Hc * Wc + C * covered
    cand = float(np.diff(ptr).astype(np.int64).sum()) * _lib.MOSAIC_TILE_H * _lib.MOSAIC_TILE_W
    return {"frames": n, "frame": [h, w], "canvas": [Hc, Wc], "canvas_mp": Hc * Wc / 1e6, "ms": ms, "GB_per_s": nbytes / ms / 1e6,
            "pct_of_hbm": 100.0 * nbytes / ms / 1e9 / HBM_TBS, "bytes": nbytes, "candidate_frame_pixels": cand,
            "covered_frame_pixels": covered, "coverage": float((mask != 0).float().mean())}


def host_time(frames, M, canvas, threads):
    import cv2
    from oracle import mosaic as OM
    cv2.setNumThreads(threads)
    t0 = time.perf_counter()
    OM.blend(frames, M, canvas[0], canvas[1], 64)
    return (time.perf_counter() - t0) * 1e3


def cli_time(root, n=8, h=1080, w=1920):
    import cv2
    import mosaic_images as cli
    _, frames, _, _ = SW.sweep(n, h, w, seed=4)
    raw = os.path.join(root, "raw")
    os.makedirs(raw)
    for k, f in enumerate(frames):
        cv2.imwrite(os.path.join(raw, "F_%03d.JPG" % k), f[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, 95])
    argv = ["--frames", raw, "--seeded_weights", "True", "--model_dir", os.path.join(root, "none")]
    res = {}
    for run in ("warm", "timed"):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        try:
            cli.main(argv + ["--out_dir", os.path.join(root, run)])
        except SystemExit as e:                               # e.g. seeded weights chaining to a canvas the encoder rejects
            return {"error": str(e)}
        torch.cuda.synchronize()
        res[run] = (time.perf_counter() - t0) * 1e3
    return {"frames": n, "frame": [h, w], "ms_per_frame": res["timed"] / n}


def multiband_bytes(M, h, w, canvas, bands):
    """Bytes the multi-band kernels move at least, from the shapes: per frame element of level i, G (4) and W (2) written
    once (base level or pyrDown) and read by pyrDown and accumulate, G_{i+1} read again for pyrUp; per canvas element of
    level i, (acc, wacc) written (8) and read (8), R_i written and read (8, i >= 1); the source pixels (3 per covered
    frame pixel) and the uint8 mosaic and mask (4 per canvas pixel)."""
    from oracle import multiband as MB
    Hc, Wc = canvas
    rois, _ = mosaic.multiband_rois(M, [(h, w)] * len(M), Hc, Wc)
    B = MB.num_bands(Hc, Wc, bands)
    a = 1 << B
    Hp, Wp = Hc + (-Hc) % a, Wc + (-Wc) % a
    frame_el = [0] * (B + 1)
    for x0, y0, x1, y1 in rois:
        r = MB.padded_rect(int(x0), int(y0), int(x1 - x0), int(y1 - y0), Hp, Wp, B)
        for i in range(B + 1):
            frame_el[i] += ((r[2] - r[0]) >> i) * ((r[3] - r[1]) >> i)
    canvas_el = [(Hp >> i) * (Wp >> i) for i in range(B + 1)]
    nbytes = 3 * sum(mapped_area(M[k], h, w) for k in range(len(M))) + 4 * Hc * Wc
    for i in range(B + 1):
        nbytes += 6 * frame_el[i] * (3 if i < B else 2) + (4 * frame_el[i + 1] if i < B else 0)
        nbytes += 16 * canvas_el[i] + (16 if i >= 1 else 0) * canvas_el[i]
    return nbytes, B, frame_el, canvas_el


def multiband_time(frames, M, canvas, bands, reps=5):
    Hc, Wc = canvas
    dev = [torch.from_numpy(f).cuda() for f in frames]
    ops.mosaic_multiband_u8(dev, M, Hc, Wc, bands)
    torch.cuda.synchronize()
    _lib.lib.udh_prof_enable(1)
    _lib.lib.udh_prof_reset()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        ops.mosaic_multiband_u8(dev, M, Hc, Wc, bands)
    e1.record()
    e1.synchronize()
    ph = _lib.prof_read_all()
    _lib.lib.udh_prof_enable(0)
    ms = e0.elapsed_time(e1) / reps
    nbytes, B, frame_el, canvas_el = multiband_bytes(M, frames[0].shape[0], frames[0].shape[1], canvas, bands)
    phases = {k.split(".")[1]: v[0] / reps for k, v in ph.items() if k.startswith("multiband.")}
    return {"frames": len(frames), "frame": list(frames[0].shape[:2]), "canvas": [Hc, Wc], "canvas_mp": Hc * Wc / 1e6,
            "bands": bands, "bands_used": B, "ms": ms, "phase_ms": phases, "bytes": nbytes, "GB_per_s": nbytes / ms / 1e6,
            "pct_of_hbm": 100.0 * nbytes / ms / 1e9 / HBM_TBS, "frame_elements": frame_el, "canvas_elements": canvas_el}


def multiband_host_time(frames, M, canvas, bands, threads):
    import cv2
    from oracle import multiband as MB
    cv2.setNumThreads(threads)
    t0 = time.perf_counter()
    fed = MB.fed(frames, M, canvas[0], canvas[1])
    t1 = time.perf_counter()
    MB.cv2_blend(*fed, canvas[0], canvas[1], bands)
    t2 = time.perf_counter()
    return {"rois_ms": (t1 - t0) * 1e3, "blender_ms": (t2 - t1) * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--legs", default="feather,multiband")
    legs = ap.parse_args().legs.split(",")
    torch.cuda.set_device(0)
    out = {"gpu": torch.cuda.get_device_name(0), "card": jpeg_time.card(), "feather": 64}
    if "multiband" in legs:
        for n, h, w in ((32, 1080, 1920), (16, 3000, 4000)):
            frames, M, canvas = placed_sweep(n, h, w)
            for bands in (5, 8):
                out["multiband_%dx%dx%d_b%d" % (n, h, w, bands)] = r = multiband_time(frames, M, canvas, bands)
                print(json.dumps(r), flush=True)
            host = {"bands": 5}
            for t in (1, 16):
                host["threads_%d" % t] = multiband_host_time(frames, M, canvas, 5, t)
            out["multiband_host_%dx%dx%d" % (n, h, w)] = host
            print(json.dumps(host), flush=True)
            del frames
    if "feather" not in legs:
        print(json.dumps(out))
        return
    for n, h, w in ((32, 1080, 1920), (16, 3000, 4000)):
        frames, M, canvas = placed_sweep(n, h, w)
        out["kernel_%dx%dx%d" % (n, h, w)] = r = kernel_time(frames, M, canvas)
        print(json.dumps(r), flush=True)
        del frames
    frames, M, canvas = placed_sweep(8, 1080, 1920)
    host = {"kernel_ms": kernel_time(frames, M, canvas)["ms"], "canvas": list(canvas)}
    for t in (1, 16):
        host["host_ms_threads_%d" % t] = host_time(frames, M, canvas, t)
    out["host_8x1080x1920"] = host
    print(json.dumps(host), flush=True)
    root = tempfile.mkdtemp(prefix="mosaic_time_")
    try:
        out["cli_8x1080x1920"] = cli_time(root)
    finally:
        shutil.rmtree(root, ignore_errors=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
