"""Image-alignment timing, in one run on the GPU:
  * end-to-end pairs/s of align_images.py's path (device decode + prep + forward + warp + JPEG encode, files written) for
    1024 pairs of 240x320 quality-95 JPEGs and for 16 pairs of 3000x4000 (12 MP) JPEGs;
  * the same pairs through a host path: cv2.imread, the loader's host normalise + cv2.resize, the same engine forward,
    cv2.warpPerspective and cv2.imencode;
  * udh_warp_perspective_u8 alone on a batch of 12 MP BGR frames: ms per frame and achieved GB/s (bytes read + written)
    against the H100 SXM's 3.35 TB/s.
The inputs are seeded textures written to a temporary directory (removed at exit).  Prints one JSON line with the card
name and power limit read in the same run.

    python tools/align_time.py [--small 1024] [--large 16]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import align_images as cli  # noqa: E402
from tools import jpeg_time  # noqa: E402
from unsuperviseddeephomographyral2018_b200 import align, dataloader as dl, ops  # noqa: E402

HBM_TBS = 3.35


def texture(rng, h, w):
    import cv2
    small = rng.integers(0, 256, (max(h // 8, 2), max(w // 8, 2), 3), np.uint8)
    img = cv2.resize(small, (w, h), interpolation=cv2.INTER_CUBIC)
    return np.clip(img.astype(np.int16) + rng.integers(-12, 13, img.shape), 0, 255).astype(np.uint8)


def write_pairs(root, n, h, w, seed):
    import cv2
    rng = np.random.default_rng(seed)
    M = np.array([[1.0, 0.03, 0.02 * w], [-0.02, 1.0, -0.015 * h], [2e-5 * 320 / w, 0, 1.0]])
    lines = []
    for k in range(n):
        a = texture(rng, h, w)
        b = cv2.warpPerspective(a, M, (w, h), borderMode=cv2.BORDER_REFLECT)
        for nm, img in (("%d_1.jpg" % k, a), ("%d_2.jpg" % k, b)):
            cv2.imwrite(os.path.join(root, nm), img, [cv2.IMWRITE_JPEG_QUALITY, 95])
        lines.append("%d_1.jpg %d_2.jpg" % (k, k))
    with open(os.path.join(root, "pairs.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
    return os.path.join(root, "pairs.txt")


def device_path(est, pairs, out_dir):
    args = cli.build_parser().parse_args(["--pairs", pairs, "--out_dir", out_dir, "--batch_size", str(est.B)])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    cli.run(args, est, align.decode_images, ops.encode_jpeg)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def host_path(est, pairs, out_dir):
    import cv2
    names, paths = align.read_pairs(pairs)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for c0 in range(0, len(paths), est.B):
        chunk = paths[c0:c0 + est.B]
        bgr = [(cv2.imread(p1, cv2.IMREAD_COLOR), cv2.imread(p2, cv2.IMREAD_COLOR)) for p1, p2 in chunk]
        planes = [np.stack([dl.normalise_resize_host(cv2.cvtColor(im[s], cv2.COLOR_BGR2RGB).astype(np.float32), est.img_h, est.img_w)
                            for im in bgr]) for s in (0, 1)]
        I_pl, Ip_pl = (torch.from_numpy(p).cuda() for p in planes)
        pts1 = torch.from_numpy(align.centred_corners(len(chunk), est.img_h, est.img_w, est.P)).cuda()
        h4p = est._forward(dl.gather_patches(I_pl, Ip_pl, I_pl, Ip_pl, pts1, est.P, est.img_w), len(chunk)).cpu().numpy()
        for j, (a, b) in enumerate(bgr):
            H = align.image_homography(h4p[j:j + 1], pts1[j:j + 1].cpu().numpy(), a.shape[:2], b.shape[:2], est.img_h, est.img_w)[0]
            ok, buf = cv2.imencode(".jpg", cv2.warpPerspective(a, H, (b.shape[1], b.shape[0])), [cv2.IMWRITE_JPEG_QUALITY, 95])
            with open(os.path.join(out_dir, "%d_warped.jpg" % (c0 + j)), "wb") as f:
                f.write(buf.tobytes())
    return time.perf_counter() - t0


def warp_alone(B=4, h=3000, w=4000, iters=20):
    rng = np.random.default_rng(1)
    src = torch.from_numpy(np.stack([texture(rng, h, w) for _ in range(B)])).cuda()
    M = torch.tensor([[0.98, 0.05, 40.0], [-0.04, 1.01, -25.0], [2e-6, -1e-5, 1.0]], dtype=torch.float64).repeat(B, 1, 1).cuda()
    for _ in range(3):
        ops.warp_perspective_u8(src, M, h, w)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.warp_perspective_u8(src, M, h, w)
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / iters
    nbytes = 2 * B * h * w * 3
    return dict(batch=B, ms_per_batch=round(ms, 4), ms_per_frame=round(ms / B, 4), GBps=round(nbytes / ms / 1e6, 1),
                share_of_hbm=round(nbytes / ms / 1e9 / HBM_TBS, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", type=int, default=1024)
    ap.add_argument("--large", type=int, default=16)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = dict(tool="align_time", card=jpeg_time.card())
    est = align.HomographyEstimator(batch_size=128, seed=0)
    tmp = tempfile.mkdtemp(prefix="align_time_")
    try:
        for tag, n, h, w in (("240x320", a.small, 240, 320), ("3000x4000", a.large, 3000, 4000)):
            root = os.path.join(tmp, tag)
            os.makedirs(os.path.join(root, "out_dev")); os.makedirs(os.path.join(root, "out_host"))
            pairs = write_pairs(root, n, h, w, seed=h)
            device_path(est, pairs, os.path.join(root, "out_dev"))           # warm-up: modules, plans, allocator
            dev = min(device_path(est, pairs, os.path.join(root, "out_dev")) for _ in range(2))
            host_path(est, pairs, os.path.join(root, "out_host"))
            host = min(host_path(est, pairs, os.path.join(root, "out_host")) for _ in range(2))
            res[tag] = dict(pairs=n, device_pairs_per_s=round(n / dev, 1), host_pairs_per_s=round(n / host, 1),
                            speedup=round(host / dev, 2), prep_paths={"%dx%d" % k: v for k, v in est.prep_paths.items()})
        res["warp_12mp_bgr"] = warp_alone()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
