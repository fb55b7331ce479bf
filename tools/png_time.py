"""PNG decode timing, in one run:
  * writes two temporary on-disk sets in the reference's layout (I/, I_prime/, list, pts1.txt, gt.txt) from the same
    device-generated 240x320 pairs: one as PNG (cv2.imwrite defaults), one as JPEG (quality 95, 4:2:0); removed at exit;
  * device PNG decode images/s per 1024-image launch (CUDA events), and the host plan's time;
  * cv2 PNG decode images/s on one host thread and on a pool of 16 threads;
  * train throughput (B = 128, h_loss, two-limb mode) fed from the PNG set, from the JPEG set, and by --synthetic, with
    the loader's decode_stats per group for the disk-fed runs.
Prints one JSON line with the card name, power limit and max SM clock read in the same run.

    python tools/png_time.py [--pairs 2048] [--steps 40]
"""
import argparse
import concurrent.futures
import json
import os
import shutil
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools import jpeg_time  # noqa: E402
from unsuperviseddeephomographyral2018_b200 import _lib, ops, synthetic  # noqa: E402


def write_sets(png_root, jpg_root, pairs, B=128):
    import cv2
    for root in (png_root, jpg_root):
        os.makedirs(os.path.join(root, "I")); os.makedirs(os.path.join(root, "I_prime"))
    names, pts1, gt = [], [], []
    for s in range(0, pairs, B):
        b = synthetic.make_batch_fast(B, seed=1000 + s)
        I, Ip = b["I_u8"].cpu().numpy(), b["I_prime_u8"].cpu().numpy()
        for j in range(min(B, pairs - s)):
            name = "%06d" % (s + j + 1)
            for sub, img in (("I", I[j]), ("I_prime", Ip[j])):
                cv2.imwrite(os.path.join(png_root, sub, name + ".png"), img[..., ::-1])      # cv2 defaults: level 1, RLE strategy
                cv2.imwrite(os.path.join(jpg_root, sub, name + ".jpg"), img[..., ::-1])
            names.append(name)
        pts1.append(b["pts1"].cpu().numpy()); gt.append(b["gt"].cpu().numpy())
    for root, ext in ((png_root, ".png"), (jpg_root, ".jpg")):
        with open(os.path.join(root, "list.txt"), "w") as f:
            f.write("\n".join("%s%s %s%s" % (n, ext, n, ext) for n in names) + "\n")
        np.savetxt(os.path.join(root, "pts1.txt"), np.concatenate(pts1)[:pairs].astype(np.float64))
        np.savetxt(os.path.join(root, "gt.txt"), np.concatenate(gt)[:pairs].astype(np.float64))


def device_decode(blobs, n=1024, reps=10):
    plan = ops.PngPlan(blobs[:n], 240, 320)
    for _ in range(2):
        out, status = plan.decode()
    assert int(status.ne(0).sum()) == 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(reps):
        plan.decode()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    t0 = time.perf_counter()
    for _ in range(3):
        ops.PngPlan(blobs[:n], 240, 320)
    return {"images": n, "ms_per_launch": ms, "images_per_s": n / (ms * 1e-3), "host_plan_ms": (time.perf_counter() - t0) / 3 * 1e3}


def host_decode(blobs, threads=16):
    import cv2
    dec = lambda b: cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
    cv2.setNumThreads(1)
    n1 = 256
    t0 = time.perf_counter()
    for b in blobs[:n1]:
        dec(b)
    one = n1 / (time.perf_counter() - t0)
    with concurrent.futures.ThreadPoolExecutor(threads) as ex:
        list(ex.map(dec, blobs[:256]))
        t0 = time.perf_counter()
        list(ex.map(dec, blobs))
        pool = len(blobs) / (time.perf_counter() - t0)
    return {"one_thread_images_per_s": one, "pool_images_per_s": pool, "pool_threads": threads, "cpu_count": os.cpu_count(),
            "cv2": cv2.__version__}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=8)
    args = ap.parse_args()
    _lib.require_device()
    png_root, jpg_root = tempfile.mkdtemp(prefix="udh_png_time_"), tempfile.mkdtemp(prefix="udh_png_time_jpg_")
    try:
        write_sets(png_root, jpg_root, args.pairs)
        names = sorted(os.listdir(os.path.join(png_root, "I")))
        blobs = []
        for n in names:
            for sub in ("I", "I_prime"):
                with open(os.path.join(png_root, sub, n), "rb") as f:
                    blobs.append(f.read())
        out = {"measurement": "PNG decode, 240x320 RGB (cv2.imwrite defaults), %d pairs on disk" % args.pairs,
               "gpu": torch.cuda.get_device_name(0), "card": jpeg_time.card(), "mean_file_bytes": float(np.mean([len(b) for b in blobs]))}
        out["device_decode"] = device_decode(blobs)
        out["host_decode"] = host_decode(blobs)
        out["train_disk_png"] = jpeg_time.train(png_root, args.pairs, args.steps, args.warmup, 0)
        out["train_disk_jpeg"] = jpeg_time.train(jpg_root, args.pairs, args.steps, args.warmup, 0)
        out["train_synthetic"] = jpeg_time.train(png_root, args.pairs, args.steps, args.warmup, args.pairs)
        out["card_after"] = jpeg_time.card()
        print(json.dumps(out))
    finally:
        shutil.rmtree(png_root, ignore_errors=True)
        shutil.rmtree(jpg_root, ignore_errors=True)


if __name__ == "__main__":
    main()
