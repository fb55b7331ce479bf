"""The reference's synthetic-dataset generator (code/utils/gen_synthetic_data.py) in Python 3, with the pixel work on the GPU.

For every raw image (sorted names, hidden files skipped): cv2.imread, cv2.resize to img_h x img_w (INTER_LINEAR),
cv2.cvtColor(..., COLOR_RGB2GRAY); then img_per_real pairs, each drawn from one random.Random(seed) in the reference's
order (y, then x, then (dx, dy) per corner TL, TR, BR, BL as four_points lists them), H = getPerspectiveTransform,
H_inverse = inv(H), and the reference's numpy_transformer of the colour and of the gray image by H_inverse.  Files follow
the reference: I/<n>.jpg and I_prime/<n>.jpg (gray only in train mode with --color false), np.savetxt rows of gt and
pts1, "<n>.jpg <n>.jpg" list lines, the num_data cutoff, test mode's start_index = num_data, and --resume N's deletions.
Unreadable files are skipped without consuming an index.

The driver (draws, names, text files, cutoffs) is shared; a backend does the pixel work.  DeviceBackend: raw images
decoded by cv2.imread on a pool of host threads (arbitrary user files: progressive JPEG and PNG included); resize, gray,
warp and JPEG encode on the GPU (udh_resize_linear_u8, udh_gen_warp_u8, udh_jpeg_encode), each bit-identical to the
host calls; files written by a background thread.  oracle/gen_data.py's HostBackend does the same with cv2 and NumPy.

Deliberate deviations from the reference: the raw list is sorted (os.listdir order is not reproducible), and `--visual`
is accepted and draws nothing.
"""
import concurrent.futures
import os
import random

import numpy as np

from . import gen_io

CHUNK = 64                     # raw images per device round


def pair_draws(rnd, rho, patch_size, height, width):
    """One pair's draws, in homographyGeneration's order -> (four_points, perturbed_four_points)."""
    y = rnd.randint(rho, height - rho - patch_size)
    x = rnd.randint(rho, width - rho - patch_size)
    four = [(x, y), (patch_size + x, y), (patch_size + x, patch_size + y), (x, patch_size + y)]
    pert = []
    for p in four:
        dx = rnd.randint(-rho, rho)
        dy = rnd.randint(-rho, rho)
        pert.append((p[0] + dx, p[1] + dy))
    return four, pert


def pair_theta(four, pert, height, width):
    """numpy_transformer's matrix for warping by H_inverse: inv(M) inv(H_inverse) M, with the reference's own expressions
    (M float32, H from cv2.getPerspectiveTransform).  None when H is singular (the reference then stops that image)."""
    import cv2
    H = cv2.getPerspectiveTransform(np.float32(four), np.float32(pert))
    try:
        H_inverse = np.linalg.inv(H)
    except np.linalg.LinAlgError:
        return None
    M = np.array([[width / 2.0, 0, width / 2.0], [0, height / 2.0, height / 2.0], [0, 0, 1.]]).astype(np.float32)
    return np.dot(np.dot(np.linalg.inv(M), np.linalg.inv(H_inverse)), M)


def raw_list(path):
    return sorted(n for n in os.listdir(path) if not n.startswith("."))


def read_raw(path):
    """cv2.imread(path) (BGR uint8) or None when cv2 cannot read it."""
    import cv2
    return cv2.imread(path)


def generate(args, backend, seed=0):
    """Run the generator with `backend` (DeviceBackend or oracle.gen_data.HostBackend); returns the next free index."""
    rnd = random.Random(seed)
    gen_io.prepare(args, (args.I_dir, args.I_prime_dir))
    names = raw_list(args.raw_data_path)
    end = args.num_data + args.start_index
    index = args.start_index
    train = args.mode == "train"
    gray_files = train and not args.color
    files = None
    writer = None if args.debug else gen_io.Writer()
    pool = concurrent.futures.ThreadPoolExecutor(min(16, os.cpu_count() or 1))
    paths = [os.path.join(args.raw_data_path, n) for n in names]
    chunks = [paths[i:i + CHUNK] for i in range(0, len(paths), CHUNK)]
    nxt = pool.map(read_raw, chunks[0]) if chunks else None
    try:
        for ci in range(len(chunks)):
            raws = list(nxt)
            nxt = pool.map(read_raw, chunks[ci + 1]) if ci + 1 < len(chunks) else None   # decode ahead
            raws = [r for r in raws if r is not None]                                  # unreadable: no index consumed
            if not raws:
                continue
            pairs = []                                       # (raw position, index, four, pert, theta)
            for k in range(len(raws)):
                if files is None and not args.debug:
                    files = [open(f, "ab") for f in ((args.pts1_file, args.gt_file, args.filenames_file) if train else
                                                     (args.test_pts1_file, args.test_gt_file, args.test_filenames_file))]
                stop = False
                for _ in range(args.img_per_real):
                    four, pert = pair_draws(rnd, args.rho, args.patch_size, args.img_h, args.img_w)
                    theta = pair_theta(four, pert, args.img_h, args.img_w)
                    if theta is None:
                        break
                    if args.debug:                           # the reference returns after one pair and writes nothing
                        index += 1
                        break
                    pairs.append((k, index, four, pert, theta))
                    index += 1
                    if index >= end:
                        stop = True
                        break
                if stop or index >= end:
                    break
            if pairs:
                blobs_i, blobs_p = backend.pairs(raws, [p[0] for p in pairs], np.stack([p[4] for p in pairs]), args.img_h,
                                                 args.img_w, gray_files)
                f_pts1, f_gt, f_list = files
                for (k, n, four, pert, _), bi, bp in zip(pairs, blobs_i, blobs_p):
                    writer.put(os.path.join(args.I_dir, "%d.jpg" % n), bi)
                    if args.I_prime_dir is not None:
                        writer.put(os.path.join(args.I_prime_dir, "%d.jpg" % n), bp)
                    gt = np.subtract(np.array(pert), np.array(four)).flatten().astype(np.float32)
                    pts1 = np.array(four).flatten().astype(np.float32)
                    np.savetxt(f_gt, [gt], delimiter=" ")
                    np.savetxt(f_pts1, [pts1], delimiter=" ")
                    f_list.write(("%d.jpg %d.jpg\n" % (n, n)).encode())
            if index >= end:
                break
    finally:
        pool.shutdown(wait=True, cancel_futures=True)
        if files:
            for f in files:
                f.close()
        if writer:
            writer.close()
    return index


class DeviceBackend:
    """Resize, gray, warp and JPEG encode on the GPU."""

    MAX_PAIRS = 1024

    def __init__(self, quality=95):
        from . import _lib
        _lib.require_device()
        self.quality = quality

    def pairs(self, raws, which, thetas, height, width, gray_files):
        """raws: decoded BGR images; which[p]: the raw image of pair p; thetas [P,3,3] float64 -> (I files, I' files)."""
        import torch
        from . import ops
        resized = torch.empty(len(raws), height, width, 3, dtype=torch.uint8, device="cuda")
        groups = {}
        for k, r in enumerate(raws):
            groups.setdefault(r.shape, []).append(k)
        for shape, ks in groups.items():                     # one launch per source size
            src = torch.from_numpy(np.stack([raws[k] for k in ks])).cuda(non_blocking=True)
            resized[torch.tensor(ks, device="cuda")] = ops.resize_linear_u8(src, height, width)
        out_i, out_p = [], []
        for p0 in range(0, len(which), self.MAX_PAIRS):        # bounded launches whatever --img_per_real is
            src = resized[torch.tensor(which[p0:p0 + self.MAX_PAIRS], device="cuda")].contiguous()
            th = torch.from_numpy(np.ascontiguousarray(thetas[p0:p0 + self.MAX_PAIRS])).cuda()
            gray, warped, warped_gray = ops.gen_warp_u8(src, th)
            a, b = (gray, warped_gray) if gray_files else (src, warped)
            out_i += ops.encode_jpeg(a, self.quality)
            out_p += ops.encode_jpeg(b, self.quality)
        return out_i, out_p


def build_parser():
    import argparse

    def str2bool(s):
        return s.lower() == "true"

    p = argparse.ArgumentParser(
        description="Generate the reference's synthetic dataset (gen_synthetic_data.py) with the pixel work on the GPU. "
                    "Deviations from the reference: raw files are taken in sorted order (os.listdir order is not "
                    "reproducible), draws come from random.Random(--seed), --visual draws nothing, and the file and "
                    "directory defaults are derived from --data_path.")
    p.add_argument("--mode", type=str, default="test", choices=["train", "test"])
    p.add_argument("--color", type=str2bool, default="true", help="Generate color or gray images (gray only in train mode)")
    p.add_argument("--debug", type=str2bool, default="false", help="Draw only: nothing deleted or stored")
    p.add_argument("--raw_data_path", type=str, default="rawdata/train/")
    p.add_argument("--test_raw_data_path", type=str, default="rawdata/test/")
    p.add_argument("--data_path", type=str, default="data/synthetic/45/")
    for name in ("I_dir", "I_prime_dir", "pts1_file", "test_pts1_file", "gt_file", "test_gt_file", "filenames_file",
                 "test_filenames_file"):
        p.add_argument("--" + name, type=str, default=None)
    p.add_argument("--num_data", type=int, default=100000)
    p.add_argument("--test_num_data", type=int, default=5000)
    p.add_argument("--visual", type=str2bool, default="false", help="Accepted; draws nothing")
    p.add_argument("--artifact_mode", type=str, default="None", choices=["noise", "None"], help="Accepted; unused, as in the reference")
    p.add_argument("--img_w", type=int, default=320)
    p.add_argument("--img_h", type=int, default=240)
    p.add_argument("--rho", type=int, default=45)
    p.add_argument("--patch_size", type=int, default=128)
    p.add_argument("--img_per_real", type=int, default=2)
    p.add_argument("--resume", type=str, default="N", help="Y: append to existing data. N: delete old data, create new data")
    p.add_argument("--start_index", type=int, default=0)
    p.add_argument("--seed", type=int, default=0, help="Seed of the random.Random that draws every pair")
    return p


def resolve_args(args):
    """Reference defaults relative to --data_path, then test mode's substitutions."""
    d = args.data_path
    defaults = dict(I_dir=os.path.join(d, "I/"), I_prime_dir=os.path.join(d, "I_prime/"), pts1_file=os.path.join(d, "pts1.txt"),
                    filenames_file=os.path.join(d, "train_synthetic.txt"), gt_file=os.path.join(d, "gt.txt"),
                    test_pts1_file=os.path.join(d, "test_pts1.txt"), test_filenames_file=os.path.join(d, "test_synthetic.txt"),
                    test_gt_file=os.path.join(d, "test_gt.txt"))
    for k, v in defaults.items():
        if getattr(args, k) is None:
            setattr(args, k, v)
    if args.mode == "test":
        args.start_index = args.num_data
        args.num_data = args.test_num_data
        args.raw_data_path = args.test_raw_data_path
    os.makedirs(d, exist_ok=True)
    return args


def main(argv=None):
    args = resolve_args(build_parser().parse_args(argv))
    n = generate(args, DeviceBackend(), seed=args.seed)
    print("generated pairs %d .. %d under %s" % (args.start_index, n - 1, args.data_path))
    return n
