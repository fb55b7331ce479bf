"""Real-data generator and camera-frame decode timing, in one run, on a seeded sequence of overlapping 12 MP frames
(4000x3000, quality 95, 4:2:0, no restart markers) written with cv2.imencode to a temporary directory:
  - device decode (JpegPlan.decode: copies of plan and data, entropy, IDCT, colour; CUDA events) of one frame and of a
    batch of 8, with the parallel entropy path on and off;
  - cv2.imread of the same files on one host thread and on a pool of 16;
  - the loader's 240x320 quality-95 files (about 30 kB, one segment) in launches of 128 and 1024, path on and off: the
    length threshold keeps them on the serial path;
  - gen_real_data.py's device generator against the host generator (oracle.gen_real_data.HostBackend) in samples/s,
    train mode with colour, with a check that the two directories are identical.
Every decode is checked against cv2 first.  Prints one JSON line with the card name, power limit and clocks read in the
same run.

    python tools/gen_real_time.py [--frames 16] [--reps 5]
"""
import argparse
import concurrent.futures
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import gen_real_data as OR  # noqa: E402
from oracle import jpeg as J  # noqa: E402
from unsuperviseddeephomographyral2018_b200 import _lib, gen_real_data, ops  # noqa: E402


def card():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=10).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "max_sm_mhz": float(out[2]), "sm_mhz_now": float(out[3]),
                "mem_mhz_now": float(out[4])}
    except Exception as e:
        return {"error": repr(e)}


def timed(fn, reps):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def set_parallel(mode):
    _lib.check(_lib.lib.udh_debug_jpeg_set_parallel(mode))


def camera_frames(root, n, seed=0):
    import cv2
    rng = np.random.default_rng(seed)
    H, W, step = 3000, 4000, 160
    small = rng.integers(0, 256, (H // 24, (W + step * n) // 24 + 1, 3), dtype=np.uint8)
    scene = cv2.resize(small, (small.shape[1] * 24, small.shape[0] * 24), interpolation=cv2.INTER_CUBIC)
    scene = cv2.add(scene, rng.integers(0, 16, scene.shape, dtype=np.uint8))
    paths = []
    for k in range(n):
        paths.append(os.path.join(root, "DSC_%04d.JPG" % (k + 1)))
        cv2.imwrite(paths[-1], np.ascontiguousarray(scene[:, step * k:step * k + W]), [cv2.IMWRITE_JPEG_QUALITY, 95])
    return paths


def parallel_segments(plan):
    import ctypes
    n = ctypes.c_int(-1)
    _lib.check(_lib.lib.udh_debug_jpeg_parallel_segments(plan.plan.data_ptr(), ctypes.c_void_p(plan.ws.data_ptr()), ctypes.byref(n)))
    return n.value


def decode_times(blobs, h, w, reps):
    """ms per JpegPlan.decode with the parallel path on (length-picked) and off, after checking both against cv2."""
    import cv2
    res = {}
    for name, mode in (("parallel", -1), ("serial", 0)):
        set_parallel(mode)
        try:
            plan = ops.JpegPlan(blobs, h, w)
        finally:
            set_parallel(-1)
        out, st = plan.decode()
        got = out.cpu().numpy()
        assert (st.cpu().numpy() == 0).all()
        for k in range(min(len(blobs), 4)):
            assert np.array_equal(got[k], cv2.imdecode(np.frombuffer(blobs[k], np.uint8), cv2.IMREAD_COLOR)[..., ::-1])
        ms = timed(plan.decode, reps if name == "parallel" or len(blobs[0]) < 100000 else 1)
        res[name] = {"ms_per_launch": ms, "images_per_s": len(blobs) / (ms * 1e-3), "parallel_segments": parallel_segments(plan)}
    return res


def generator(raw, root):
    res = {}
    for side, backend in (("device", gen_real_data.DeviceBackend()), ("host", OR.HostBackend())):
        data = os.path.join(root, side) + "/"
        argv = ["--mode", "train", "--raw_data_path", raw, "--data_path", data, "--num_data", "100000", "--seed", "0"]
        args = gen_real_data.resolve_args(gen_real_data.build_parser().parse_args(argv))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n = gen_real_data.generate(args, backend, seed=0)
        wall = time.perf_counter() - t0
        res[side] = {"samples": n, "frames": len(gen_real_data.frame_list(raw)), "wall_s": wall, "samples_per_s": n / wall,
                     "pairs_per_s": (len(gen_real_data.frame_list(raw)) - 1) / wall}
    same = True
    for d in ("I", "I_prime", "FULL_I", "FULL_I_prime"):
        for f in os.listdir(os.path.join(root, "host", d)):
            same &= open(os.path.join(root, "device", d, f), "rb").read() == open(os.path.join(root, "host", d, f), "rb").read()
    for f in ("pts1.txt", "train_real.txt"):
        same &= open(os.path.join(root, "device", f), "rb").read() == open(os.path.join(root, "host", f), "rb").read()
    res["directories_identical"] = bool(same)
    return res


def main():
    import cv2
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    _lib.require_device()
    out = {"measurement": "camera-frame decode (12 MP q95 4:2:0) and gen_real_data.py device vs host", "gpu": torch.cuda.get_device_name(0),
           "card_before": card(), "cpu_count": os.cpu_count()}
    root = tempfile.mkdtemp(prefix="udh_gen_real_time_")
    try:
        raw = os.path.join(root, "raw")
        os.makedirs(raw)
        paths = camera_frames(raw, args.frames)
        blobs = [open(p, "rb").read() for p in paths]
        out["frame_bytes_mean"] = float(np.mean([len(b) for b in blobs]))
        out["decode_12mp_N=1"] = decode_times(blobs[:1], 3000, 4000, args.reps)
        out["decode_12mp_N=8"] = decode_times(blobs[:8], 3000, 4000, args.reps)
        cv2.setNumThreads(1)
        t0 = time.perf_counter()
        for p in paths[:8]:
            cv2.imread(p)
        out["cv2_imread_12mp_one_thread_ms"] = (time.perf_counter() - t0) * 1e3 / 8
        with concurrent.futures.ThreadPoolExecutor(16) as ex:
            list(ex.map(cv2.imread, paths[:4]))
            t0 = time.perf_counter()
            list(ex.map(cv2.imread, paths))
            out["cv2_imread_12mp_16_threads_images_per_s"] = len(paths) / (time.perf_counter() - t0)
        loader = []
        rng = np.random.default_rng(1)
        for k in range(1024):                                 # the loader's files: 240x320 q95 4:2:0 textures
            img = J.textured(rng, 240, 320, 3)
            loader.append(cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes())
        out["loader_file_bytes_mean"] = float(np.mean([len(b) for b in loader]))
        for n in (128, 1024):
            res = {}
            for name, mode in (("serial (length-picked)", -1), ("parallel (forced)", 1)):
                set_parallel(mode)
                try:
                    plan = ops.JpegPlan(loader[:n], 240, 320)
                finally:
                    set_parallel(-1)
                o, st = plan.decode()
                assert (st.cpu().numpy() == 0).all()
                assert np.array_equal(o[0].cpu().numpy(), cv2.imdecode(np.frombuffer(loader[0], np.uint8), cv2.IMREAD_COLOR)[..., ::-1])
                ms = timed(plan.decode, args.reps * 4)
                res[name] = {"ms_per_launch": ms, "images_per_s": n / (ms * 1e-3), "parallel_segments": parallel_segments(plan)}
            out["decode_240x320_N=%d" % n] = res
        out["generator_train_colour"] = generator(raw, root)
    finally:
        shutil.rmtree(root, ignore_errors=True)
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
