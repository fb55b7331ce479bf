"""Timing of the report images (--save_visual), B = 128 pairs of 240x320 noise images (the worst case for JPEG), in one
run:
  * render: ops.draw_report_u8 (tables, canvas fill, primitives), CUDA events over repeated launches;
  * encode: ops.encode_jpeg_device on the 240x640 canvases (quality 95), CUDA events;
  * the whole report path per batch as the harnesses run it: report.render + report.write (vertices on the host, render,
    encode, device-to-host copy, one file per image into a temporary directory), host clock after a device synchronise;
  * the host cv2 composition (the reference's drawing sequence + cv2.imencode) on 1 thread and on 16 threads.
Prints one JSON line with the card name and power limit read in the same run.

    python tools/report_time.py [--batch 128] [--reps 20]
"""
import argparse
import concurrent.futures
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import draw as D  # noqa: E402
from unsuperviseddeephomographyral2018_b200 import _lib, ops, report  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def events_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    _lib.require_device()
    import cv2
    B, h, w = a.batch, 240, 320
    rng = np.random.default_rng(0)
    I_np = rng.integers(0, 256, (B, h, w, 3), np.uint8)
    Ip_np = rng.integers(0, 256, (B, h, w, 3), np.uint8)
    c1 = rng.uniform(40, 280, (B, 4, 2)).astype(np.float32)
    c2 = (c1 + rng.normal(0, 10, (B, 4, 2))).astype(np.float32)
    pr = (c2 + rng.normal(0, 3, (B, 4, 2))).astype(np.float32)
    batch = dict(I_u8=torch.from_numpy(I_np).cuda(), I_prime_u8=torch.from_numpy(Ip_np).cuda(), aug=None)
    verts = torch.from_numpy(np.stack([report.report_vertices(x, y, z, w) for x, y, z in zip(c1, c2, pr)])).cuda()

    render_ms = events_ms(lambda: ops.draw_report_u8(batch["I_u8"], batch["I_prime_u8"], None, verts, False), a.reps)
    canv = ops.draw_report_u8(batch["I_u8"], batch["I_prime_u8"], None, verts, False)
    encode_ms = events_ms(lambda: ops.encode_jpeg_device(canv, 95), a.reps)

    with tempfile.TemporaryDirectory() as d:
        names = ["%d_loss_1.0.jpg" % k for k in range(B)]
        devnull = open(os.devnull, "w")
        stdout, sys.stdout = sys.stdout, devnull                   # report.write prints one line per file
        try:
            report.write(report.render(batch, range(B), c1, c2, pr, False), names, d)
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(5):
                report.write(report.render(batch, range(B), c1, c2, pr, False), names, d)
            torch.cuda.synchronize()
            path_ms = (time.perf_counter() - t) * 1e3 / 5
            t = time.perf_counter()
            for _ in range(5):
                vs = np.stack([report.report_vertices(x, y, z, w) for x, y, z in zip(c1, c2, pr)])
            vert_ms = (time.perf_counter() - t) * 1e3 / 5
        finally:
            sys.stdout = stdout
            devnull.close()
        assert vs.shape == (B, 20, 2)

    # host: the reference's composition and encode, per sample (denorm is not included: it is the same lookup either way)
    cv2.setNumThreads(1)

    def host_one(k):
        out = D.cv2_compose(I_np[k], Ip_np[k], c1[k], c2[k], pr[k])
        return len(cv2.imencode(".jpg", out)[1])

    host_one(0)
    t = time.perf_counter()
    for k in range(B):
        host_one(k)
    host1_ms = (time.perf_counter() - t) * 1e3
    with concurrent.futures.ThreadPoolExecutor(16) as ex:
        list(ex.map(host_one, range(16)))
        t = time.perf_counter()
        list(ex.map(host_one, range(B)))
        host16_ms = (time.perf_counter() - t) * 1e3

    print(json.dumps(dict(card=card(), batch=B, image="240x320 noise pair -> 240x640 canvas", render_ms=round(render_ms, 4),
                          encode_ms=round(encode_ms, 4), vertices_host_ms=round(vert_ms, 3), report_path_ms=round(path_ms, 3),
                          host_cv2_1thread_ms=round(host1_ms, 2), host_cv2_16threads_ms=round(host16_ms, 2), cpu_count=os.cpu_count())))


if __name__ == "__main__":
    main()
