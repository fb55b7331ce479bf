"""The reference's real-data generator (code/utils/gen_real_data.py) in Python 3, with the pixel work on the GPU.

Frames are glob(raw_path/*.JPG) (case-sensitive), sorted; frames k and k+1 form a pair, skipped when int(path[-8:-4]) of
frame k is in the mode's ignore list.  Each frame is cv2.resize'd (INTER_LINEAR) to full_img_h x full_img_w and to
img_h x img_w.  Every accepted pair gives im_per_im samples: x = randint(rho, img_w - rho - patch_size),
y = (img_h - patch_size) // 2 (Python 2's integer division), pts1 = [x,y, P+x,y, P+x,P+y, x,P+y] through np.savetxt as
float32, I/<n>.jpg, FULL_I/<n>.jpg (frame k), I_prime/<n>.jpg, FULL_I_prime/<n>.jpg (frame k + 1) as cv2.imwrite writes
them, a list line "<n>.jpg <n>.jpg", and the cutoff at start_index + num_data.  Test mode: start_index = num_data,
num_data = test_num_data, the test raw path, and a test_gt.txt row hstack(corr1.flatten(), corr2.flatten()) per sample,
where pair k takes rows 4k .. 4k+3 (frame position, ignored pairs counted) of the labels' concatenated all_corr1 /
all_corr2.  The text files are opened 'wb' at the start of every run, so each run truncates them, --resume Y included.
--resume N in train mode tries to delete gt_file first; this generator never writes one, so normally nothing is deleted
(as in the reference), and FULL_I* are never deleted.  --debug stops after the first sample and writes nothing;
--visual and --artifact_mode are accepted and do nothing.

The driver (draws, names, text files, cutoffs, --resume) is shared; a backend does the pixel work.  DeviceBackend decodes
each frame once on the GPU (udh_jpeg_decode; long entropy segments take its parallel path), flips RGB to cv2's BGR,
resizes to both sizes, takes the gray planes with the generator's gray rule and encodes each frame once per size: the
same bytes are written under every sample index that uses the frame.  Frames the device decoder does not take
(progressive, EXIF orientation other than 1, ...) are read by cv2.imread on a pool of host threads.
oracle/gen_real_data.py's HostBackend does the same with cv2.

Deliberate deviations from the reference: draws come from random.Random(--seed); the frame list is sorted with Python 3's
str order; text is written as Python 3 bytes; the five label files the reference hard-codes under
<test raw path>/labels/ are the default of --test_labels; `--mode train --color false` writes the gray images the
reference meant to (it raises NameError on full_I_gray): cvtColor(full_I, COLOR_RGB2GRAY) on BGR data, the reference's
rule everywhere else.
"""
import concurrent.futures
import glob
import os
import random

import numpy as np

from . import gen_io

TRAIN_IGNORE = [59, 60, 91, 121, 122, 149, 150, 180, 181, 238, 239, 266, 267, 296, 297, 327]
TEST_IGNORE = [30, 31]
LABEL_FILES = ["corresponences0_10.mat", "correspondences11_21.mat", "correspondences22_30.mat", "correspondences31_40.mat",
               "correspondences41_49.mat"]
FRAMES_PER_ROUND = 16            # frames decoded, resized and encoded per backend call


def frame_list(path):
    return sorted(glob.glob(os.path.join(path, "*.JPG")))


def frame_id(path):
    return int(path[len(path) - 8:len(path) - 4])


def load_labels(files):
    """query_gt_test_set: all_corr1 / all_corr2 of every .mat file, concatenated in order."""
    import scipy.io as io
    c1, c2 = [], []
    for f in files:
        m = io.loadmat(f)
        c1.append(m["all_corr1"])
        c2.append(m["all_corr2"])
    return np.concatenate(c1, axis=0), np.concatenate(c2, axis=0)


def read_frame(path):
    """cv2.imread(path): BGR uint8, or None when cv2 cannot read it."""
    import cv2
    return cv2.imread(path)


def generate(args, backend, seed=0):
    """Run the generator with `backend` (DeviceBackend or oracle.gen_real_data.HostBackend); returns the next free index."""
    rnd = random.Random(seed)
    gen_io.prepare(args, (args.I_dir, args.I_prime_dir, args.full_I_dir, args.full_I_prime_dir))
    train = args.mode == "train"
    files = None
    if not args.debug:
        names = (args.pts1_file, args.filenames_file) if train else (args.test_pts1_file, args.test_filenames_file, args.test_gt_file)
        files = [open(f, "wb") for f in names]
    writer = None
    try:
        corr1_array, corr2_array = load_labels(args.test_labels) if not train else (None, None)
        frames = frame_list(args.raw_data_path)
        P, end, index = args.patch_size, args.start_index + args.num_data, args.start_index
        samples = []                                           # (pair k, index, four_points, test_gt row or None)
        for k in range(len(frames) - 1):
            if frame_id(frames[k]) in args.ignore_list:
                continue
            corr = None
            if not train:
                corr1 = corr1_array[k * 4:k * 4 + 4].reshape([4, 2])
                corr2 = corr2_array[k * 4:k * 4 + 4].reshape([4, 2])
                corr = np.hstack([corr1.flatten(), corr2.flatten()])
            for _ in range(args.im_per_im):
                x = rnd.randint(args.rho, args.img_w - args.rho - P)
                y = (args.img_h - P) // 2
                if args.debug:                                 # the reference returns here, before any file is written
                    return index + 1
                samples.append((k, index, [(x, y), (P + x, y), (P + x, P + y), (x, P + y)], corr))
                index += 1
                if index >= end:
                    break
            if index >= end:
                break
        writer = gen_io.Writer()
        gray = train and not args.color
        pairs = {}                                             # pair k -> its samples, in order
        for smp in samples:
            pairs.setdefault(smp[0], []).append(smp)
        order, cache, i = list(pairs), {}, 0
        while i < len(order):                                  # each frame decoded once: the last one carries over
            j, need = i, set()
            while j < len(order) and len(need) < FRAMES_PER_ROUND:
                need |= {order[j], order[j] + 1}
                j += 1
            cache = {f: v for f, v in cache.items() if f in need}
            missing = sorted(need - set(cache))
            cache.update(zip(missing, backend.frames([frames[f] for f in missing], (args.img_h, args.img_w),
                                                     (args.full_img_h, args.full_img_w), gray)))
            for k in order[i:j]:
                _write_pair(args, writer, files, pairs[k], cache[k], cache[k + 1], train)
            i = j
        return index
    finally:
        if files:
            for f in files:
                f.close()
        if writer:
            writer.close()


def _write_pair(args, writer, files, samples, frame_i, frame_p, train):
    """The files and text rows of one pair's samples; frame_i / frame_p: (img_h x img_w file, full-size file)."""
    (small_i, full_i), (small_p, full_p) = frame_i, frame_p
    for _, n, four, corr in samples:
        name = "%d.jpg" % n
        writer.put(os.path.join(args.I_dir, name), small_i)
        writer.put(os.path.join(args.full_I_dir, name), full_i)
        if args.I_prime_dir is not None:
            writer.put(os.path.join(args.I_prime_dir, name), small_p)
            writer.put(os.path.join(args.full_I_prime_dir, name), full_p)
        np.savetxt(files[0], [np.array(four).flatten().astype(np.float32)], delimiter=" ")
        if not train:
            np.savetxt(files[2], [corr], delimiter=" ")
        files[1].write(("%s %s\n" % (name, name)).encode())


class DeviceBackend:
    """Decode, resize, gray and JPEG encode on the GPU; frames the device decoder does not take are read by cv2."""

    DECODE_BUDGET = 2 << 30       # device bytes one decode launch may use (a 12 MP frame: about 150 MB)

    def __init__(self, quality=95):
        from . import _lib
        _lib.require_device()
        self.quality = quality
        self.pool = concurrent.futures.ThreadPoolExecutor(min(16, os.cpu_count() or 1))

    def _decode(self, paths):
        """-> one uint8 BGR CUDA tensor [h,w,3] per path."""
        import torch
        from . import _lib, ops
        blobs = list(self.pool.map(lambda p: open(p, "rb").read(), paths))
        out, host, groups = [None] * len(paths), [], {}
        for k, b in enumerate(blobs):
            info = ops.jpeg_parse(b)
            if info.reason == 0:
                groups.setdefault((info.height, info.width), []).append(k)
            else:
                host.append(k)
        futs = {k: self.pool.submit(read_frame, paths[k]) for k in host}      # overlaps the device decode
        for (h, w), ks in groups.items():                                       # one plan per frame size
            per = _lib.lib.udh_jpeg_workspace_bytes(1, h, w) + 3 * h * w + max(len(blobs[k]) for k in ks)
            step = max(1, int(self.DECODE_BUDGET // per))
            for k0 in range(0, len(ks), step):
                sub = ks[k0:k0 + step]
                rgb, status = ops.JpegPlan([blobs[k] for k in sub], h, w).decode()
                st = status.cpu().numpy()
                for j, k in enumerate(sub):
                    if st[j]:                                  # damaged data: cv2 decides, as the reference's imread would
                        futs[k] = self.pool.submit(read_frame, paths[k])
                    else:
                        out[k] = rgb[j].flip(-1)
        for k, f in futs.items():
            im = f.result()
            if im is None:
                raise IOError("cannot read %s" % paths[k])
            out[k] = torch.from_numpy(im).cuda()
        return out

    def frames(self, paths, size, full_size, gray):
        """-> [(img_h x img_w file, full_img_h x full_img_w file)] per path: cv2.imwrite's bytes of cv2.resize(imread(path))
        at both sizes (gray: of cvtColor(..., COLOR_RGB2GRAY) applied to them)."""
        import torch
        from . import ops
        bgr = self._decode(paths)
        outs = [[None, None] for _ in paths]
        groups = {}
        for k, im in enumerate(bgr):
            groups.setdefault(tuple(im.shape), []).append(k)
        for shape, ks in groups.items():
            src = torch.stack([bgr[k] for k in ks]).contiguous()
            for s, (h, w) in enumerate((size, full_size)):
                r = ops.resize_linear_u8(src, h, w)
                files = ops.encode_jpeg(ops.gray_u8(r) if gray else r, self.quality)
                for k, f in zip(ks, files):
                    outs[k][s] = f
        return [tuple(o) for o in outs]


def build_parser():
    import argparse

    def str2bool(s):
        return s.lower() == "true"

    p = argparse.ArgumentParser(
        description="Generate the reference's real-data set (gen_real_data.py) from frame sequences with the pixel work on "
                    "the GPU.  Deviations from the reference: draws come from random.Random(--seed), --test_labels names "
                    "the label files, --mode train --color false writes gray images (the reference raises NameError), "
                    "and the file and directory defaults are derived from --data_path.")
    p.add_argument("--mode", type=str, default="train", choices=["train", "test"])
    p.add_argument("--color", type=str2bool, default="true", help="Generate color or gray images (gray only in train mode)")
    p.add_argument("--debug", type=str2bool, default="false", help="Draw only: nothing deleted or stored")
    p.add_argument("--raw_data_path", type=str, default="rawdata/real/train/", help="Frames: <raw_data_path>/*.JPG")
    p.add_argument("--test_raw_data_path", type=str, default="rawdata/real/test/")
    p.add_argument("--test_labels", type=str, nargs="+", default=None,
                   help=".mat files holding all_corr1 / all_corr2 (default: the reference's five files under "
                        "<test_raw_data_path>/labels/)")
    p.add_argument("--data_path", type=str, default="data/real/24/")
    for name in ("I_dir", "I_prime_dir", "full_I_dir", "full_I_prime_dir", "pts1_file", "test_pts1_file", "gt_file",
                 "test_gt_file", "filenames_file", "test_filenames_file"):
        p.add_argument("--" + name, type=str, default=None)
    p.add_argument("--num_data", type=int, default=10000)
    p.add_argument("--im_per_im", type=int, default=20, help="Samples per accepted pair of frames")
    p.add_argument("--test_num_data", type=int, default=1000)
    p.add_argument("--visual", type=str2bool, default="false", help="Accepted; draws nothing")
    p.add_argument("--artifact_mode", type=str, default="None", choices=["noise", "None"], help="Accepted; unused, as in the reference")
    p.add_argument("--img_w", type=int, default=190)
    p.add_argument("--img_h", type=int, default=142)
    p.add_argument("--full_img_w", type=int, default=640)
    p.add_argument("--full_img_h", type=int, default=480)
    p.add_argument("--rho", type=int, default=24)
    p.add_argument("--patch_size", type=int, default=128)
    p.add_argument("--resume", type=str, default="N", help="Y: append to existing data. N: delete old data, create new data")
    p.add_argument("--start_index", type=int, default=0)
    p.add_argument("--seed", type=int, default=0, help="Seed of the random.Random that draws every sample")
    return p


def resolve_args(args):
    """Reference defaults relative to --data_path, the ignore list, then test mode's substitutions."""
    d = args.data_path
    defaults = dict(I_dir=os.path.join(d, "I/"), I_prime_dir=os.path.join(d, "I_prime/"), full_I_dir=os.path.join(d, "FULL_I/"),
                    full_I_prime_dir=os.path.join(d, "FULL_I_prime/"), pts1_file=os.path.join(d, "pts1.txt"),
                    filenames_file=os.path.join(d, "train_real.txt"), gt_file=os.path.join(d, "gt.txt"),
                    test_pts1_file=os.path.join(d, "test_pts1.txt"), test_filenames_file=os.path.join(d, "test_real.txt"),
                    test_gt_file=os.path.join(d, "test_gt.txt"))
    for k, v in defaults.items():
        if getattr(args, k) is None:
            setattr(args, k, v)
    if args.test_labels is None:
        args.test_labels = [os.path.join(args.test_raw_data_path, "labels", f) for f in LABEL_FILES]
    args.ignore_list = TRAIN_IGNORE
    if args.mode == "test":
        args.start_index = args.num_data
        args.num_data = args.test_num_data
        args.raw_data_path = args.test_raw_data_path
        args.ignore_list = TEST_IGNORE
    os.makedirs(d, exist_ok=True)
    return args


def main(argv=None):
    args = resolve_args(build_parser().parse_args(argv))
    n = generate(args, DeviceBackend(), seed=args.seed)
    print("generated samples %d .. %d under %s" % (args.start_index, n - 1, args.data_path))
    return n
