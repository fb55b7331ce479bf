"""Dataset-generator timing, in one run: the device generator (gen_synthetic_data.py) against the host generator
(oracle.gen_data.HostBackend: cv2.resize, the NumPy warp, cv2.imencode) in pairs/s on a seeded raw set of COCO-sized
JPEGs written to a temporary directory (train mode, colour, 2 pairs per raw image), with the time split into host decode,
device work and file writes; then device encode (ops.encode_jpeg_device, CUDA events around the launch) at
N = 1, 64, 256 and 1024 images of 240x320 BGR, quality 95, against cv2.imencode on one host thread and on a pool of 16;
every device file is checked byte for byte against cv2's first.  Also the INTER_LINEAR resize 480x640 -> 240x320.
Prints one JSON line with the card name, power limit and max SM clock read in the same run.

    python tools/gen_time.py [--raw 256] [--reps 20]
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

from oracle import gen_data as OG  # noqa: E402
from oracle import jpeg_enc as E  # noqa: E402
from unsuperviseddeephomographyral2018_b200 import _lib, gen_data, ops  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=10).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "max_sm_mhz": float(out[2])}
    except Exception as e:
        return {"error": repr(e)}


def timed(fn, reps):
    for _ in range(2):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


class _Timed:
    """Wraps a backend and adds up the seconds its pairs() call takes (device work incl. copies, ending in a sync)."""

    def __init__(self, inner):
        self.inner, self.s = inner, 0.0

    def pairs(self, *a):
        t0 = time.perf_counter()
        out = self.inner.pairs(*a)
        torch.cuda.synchronize()
        self.s += time.perf_counter() - t0
        return out


def generator(nraw):
    import cv2
    rng = np.random.default_rng(0)
    root = tempfile.mkdtemp(prefix="udh_gen_time_")
    try:
        raw = os.path.join(root, "raw")
        os.makedirs(raw)
        sizes = [(480, 640), (640, 427), (375, 500), (427, 640), (640, 480)]
        for k in range(nraw):
            h, w = sizes[k % len(sizes)]
            yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
            img = np.stack([128 + 70 * np.sin(xx / (5 + 3 * c + k % 7)) * np.cos(yy / (8 + c)) for c in range(3)], -1)
            img = np.clip(img + rng.normal(0, 10, img.shape), 0, 255).astype(np.uint8)
            cv2.imwrite(os.path.join(raw, "%06d.jpg" % k), img)
        res = {}
        for side, backend in (("device", gen_data.DeviceBackend()), ("host", OG.HostBackend())):
            data = os.path.join(root, side) + "/"
            argv = ["--mode", "train", "--raw_data_path", raw, "--data_path", data, "--num_data", str(2 * nraw), "--seed", "0"]
            args = gen_data.resolve_args(gen_data.build_parser().parse_args(argv))
            tb = _Timed(backend)
            t0 = time.perf_counter()
            n = gen_data.generate(args, tb, seed=0)
            wall = time.perf_counter() - t0
            res[side] = {"pairs": n, "wall_s": wall, "pairs_per_s": n / wall, "pixel_work_s": tb.s}
        t0 = time.perf_counter()
        list(map(gen_data.read_raw, [os.path.join(raw, f) for f in sorted(os.listdir(raw))]))
        res["host_decode_one_thread_s"] = time.perf_counter() - t0
        same = all(open(os.path.join(root, "device", d, f), "rb").read() == open(os.path.join(root, "host", d, f), "rb").read()
                   for d in ("I", "I_prime") for f in os.listdir(os.path.join(root, "host", d)))
        res["directories_identical"] = bool(same)
        return res
    finally:
        shutil.rmtree(root, ignore_errors=True)


def main():
    import cv2
    ap = argparse.ArgumentParser()
    ap.add_argument("--raw", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    _lib.require_device()
    gen = generator(args.raw)
    imgs = np.stack([E.image("texture" if k % 4 else "noise", 240, 320, 3, seed=k) for k in range(1024)])
    enc = lambda im: cv2.imencode(".jpg", im, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes()
    ref = [enc(im) for im in imgs]
    got = ops.encode_jpeg(imgs, 95)
    assert got == ref, "device files differ from cv2.imencode"
    dev = torch.from_numpy(imgs).cuda()
    out = {"measurement": "dataset generator (device vs host), then baseline-JPEG encode of 240x320 BGR at quality 95 (3/4 smooth texture, 1/4 uniform noise)",
           "gpu": torch.cuda.get_device_name(0), "card": card(), "mean_file_bytes": float(np.mean([len(b) for b in ref]))}
    d = {}
    for n in (1, 64, 256, 1024):
        ms = timed(lambda: ops.encode_jpeg_device(dev[:n], 95), args.reps)
        d["N=%d" % n] = {"ms_per_launch": ms, "images_per_s": n / (ms * 1e-3)}
    out["generator"] = gen
    out["device_encode"] = d
    t0 = time.perf_counter()
    files = ops.encode_jpeg(dev[:256], 95)
    out["encode_jpeg_to_bytes_N=256_ms"] = (time.perf_counter() - t0) * 1e3
    assert files == ref[:256]
    cv2.setNumThreads(1)
    t0 = time.perf_counter()
    for im in imgs[:256]:
        enc(im)
    out["cv2_one_thread_images_per_s"] = 256 / (time.perf_counter() - t0)
    with concurrent.futures.ThreadPoolExecutor(16) as ex:
        list(ex.map(enc, imgs[:64]))
        t0 = time.perf_counter()
        list(ex.map(enc, imgs))
        out["cv2_16_threads_images_per_s"] = len(imgs) / (time.perf_counter() - t0)
    out["cpu_count"] = os.cpu_count()
    big = torch.randint(0, 256, (256, 480, 640, 3), dtype=torch.uint8, device="cuda")
    ms = timed(lambda: ops.resize_linear_u8(big, 240, 320), args.reps)
    out["resize_linear_480x640_to_240x320_N=256"] = {"ms_per_launch": ms, "images_per_s": 256 / (ms * 1e-3)}
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
