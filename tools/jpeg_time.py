"""Baseline-JPEG decode timing, in one run:
  * writes a temporary on-disk set in the reference's layout (I/, I_prime/, list, pts1.txt, gt.txt) from the device
    generator + cv2.imwrite (quality 95, 4:2:0, 240x320), removed at exit;
  * device decode images/s at N = 256 and N = 1024 (CUDA events; entropy kernel with 32 and with 1 lane per image);
  * cv2 decode images/s on one host thread and on a pool of os.cpu_count() threads;
  * train throughput (B = 128, h_loss, two-limb mode) fed from that set through Dataloader with the device decoder and
    with the host decoder only, and fed by --synthetic; for the disk-fed runs, the loader's decode_stats per group
    (reader-thread time, time next_batch waited for the reader, time next_batch spent building the group).
Prints one JSON line with the card name and power limit read in the same run.

    python tools/jpeg_time.py [--pairs 2048] [--steps 40]
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

from unsuperviseddeephomographyral2018_b200 import _lib, dataloader, engine, ops, synthetic  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=10).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "max_sm_mhz": float(out[2])}
    except Exception as e:   # the card name from torch is still reported
        return {"error": repr(e)}


def write_dataset(root, pairs, B=128):
    import cv2
    os.makedirs(os.path.join(root, "I")); os.makedirs(os.path.join(root, "I_prime"))
    names, pts1, gt = [], [], []
    for s in range(0, pairs, B):
        b = synthetic.make_batch_fast(B, seed=1000 + s)
        I, Ip = b["I_u8"].cpu().numpy(), b["I_prime_u8"].cpu().numpy()
        for j in range(min(B, pairs - s)):
            name = "%06d.jpg" % (s + j + 1)
            cv2.imwrite(os.path.join(root, "I", name), I[j][..., ::-1])          # cv2 defaults: quality 95, 4:2:0
            cv2.imwrite(os.path.join(root, "I_prime", name), Ip[j][..., ::-1])
            names.append("%s %s" % (name, name))
        pts1.append(b["pts1"].cpu().numpy()); gt.append(b["gt"].cpu().numpy())
    with open(os.path.join(root, "list.txt"), "w") as f:
        f.write("\n".join(names) + "\n")
    np.savetxt(os.path.join(root, "pts1.txt"), np.concatenate(pts1)[:pairs].astype(np.float64))
    np.savetxt(os.path.join(root, "gt.txt"), np.concatenate(gt)[:pairs].astype(np.float64))


def device_decode(blobs, n, reps=10):
    plan = ops.JpegPlan(blobs[:n], 240, 320)
    res = {}
    for lanes in (32, 1):
        _lib.check(_lib.lib.udh_debug_jpeg_set_lanes(lanes))
        for _ in range(2):
            plan.decode()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record()
        for _ in range(reps):
            plan.decode()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        res["lanes_%d" % lanes] = {"ms_per_launch": ms, "images_per_s": n / (ms * 1e-3)}
    _lib.check(_lib.lib.udh_debug_jpeg_set_lanes(32))
    t0 = time.perf_counter()
    for _ in range(reps):
        ops.JpegPlan(blobs[:n], 240, 320)
    res["host_plan_ms"] = (time.perf_counter() - t0) / reps * 1e3
    return res


def host_decode(blobs):
    import cv2
    dec = lambda b: cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
    cv2.setNumThreads(1)
    n1 = 256
    t0 = time.perf_counter()
    for b in blobs[:n1]:
        dec(b)
    one = n1 / (time.perf_counter() - t0)
    cores = os.cpu_count()
    with concurrent.futures.ThreadPoolExecutor(cores) as ex:
        list(ex.map(dec, blobs[:256]))
        t0 = time.perf_counter()
        list(ex.map(dec, blobs))
        pool = len(blobs) / (time.perf_counter() - t0)
    return {"one_thread_images_per_s": one, "pool_images_per_s": pool, "pool_threads": cores, "cpu_count": cores,
            "cv2": cv2.__version__}


def train(root, pairs, steps, warmup, synthetic_pairs, host_only=False):
    B = 128
    prm = dataloader.dataloader_params(data_path=root, filenames_file=os.path.join(root, "list.txt"), pts1_file=os.path.join(root, "pts1.txt"),
                                       gt_file=os.path.join(root, "gt.txt"), mode="train", batch_size=B, img_h=240, img_w=320,
                                       patch_size=128, augment_list=["normalize"], do_augment=0.5)
    dl = dataloader.Dataloader(prm, shuffle=True, synthetic_pairs=synthetic_pairs, seed=0)
    real_parse = ops.jpeg_parse
    if host_only:                                  # every file rejected: the loader decodes all of them with cv2.imread
        def reject(blob):
            info = _lib.JpegInfo(); info.reason = _lib.JPEG_R["NOT_JPEG"]
            return info
        ops.jpeg_parse = reject
    try:
        return _train(dl, steps, warmup, B)
    finally:
        ops.jpeg_parse = real_parse


def _train(dl, steps, warmup, B):
    eng = engine.HomographyEngine(B, numeric="bf16x3", seed=0, loss_type="h_loss", lr=5e-4)
    for _ in range(warmup):
        eng.train_step(dl.next_batch())
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    s0 = dict(dl.decode_stats)
    for _ in range(steps):
        eng.train_step(dl.next_batch())
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) / steps * 1e3
    out = {"ms_per_step": ms, "pairs_per_s": B / (ms * 1e-3)}
    st = {k: dl.decode_stats[k] - s0[k] for k in s0}
    if st["groups"]:
        g = st["groups"]
        out["per_group"] = {"batches": dl.DECODE_BATCHES, "groups_timed": g, "reader_ms": st["read_s"] / g * 1e3,
                            "wait_for_reader_ms": st["wait_s"] / g * 1e3, "build_group_ms": st["group_s"] / g * 1e3,
                            "device_images": st["device_images"] / g, "host_images": st["host_images"] / g}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=8)
    args = ap.parse_args()
    _lib.require_device()
    root = tempfile.mkdtemp(prefix="udh_jpeg_time_")
    try:
        write_dataset(root, args.pairs)
        names = sorted(os.listdir(os.path.join(root, "I")))
        blobs = []
        for n in names:
            for sub in ("I", "I_prime"):
                with open(os.path.join(root, sub, n), "rb") as f:
                    blobs.append(f.read())
        out = {"measurement": "baseline-JPEG decode, 240x320 quality 95 4:2:0 (cv2.imwrite defaults), %d pairs on disk" % args.pairs,
               "gpu": torch.cuda.get_device_name(0), "card": card(), "mean_file_bytes": float(np.mean([len(b) for b in blobs]))}
        out["device_decode"] = {"N=256": device_decode(blobs, 256), "N=1024": device_decode(blobs, 1024)}
        out["host_decode"] = host_decode(blobs)
        out["train_disk"] = train(root, args.pairs, args.steps, args.warmup, 0)
        out["train_disk_host_decode"] = train(root, args.pairs, max(8, args.steps // 4), 4, 0, host_only=True)
        out["train_synthetic"] = train(root, args.pairs, args.steps, args.warmup, args.pairs)
        out["card_after"] = card()
        print(json.dumps(out))
    finally:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
