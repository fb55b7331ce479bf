#!/usr/bin/env python
"""Align image pairs with a trained model: the homography from image 1 to image 2 of every pair, and image 1 warped into
image 2's frame (unsuperviseddeephomographyral2018_b200.align states the coordinate convention).

    python align_images.py --img1 a.jpg --img2 b.jpg --model_dir ../models/synthetic_models/
    python align_images.py --pairs pairs.txt --img_h 142 --img_w 190 --out_dir aligned/

--pairs FILE holds one `img1 img2` per line, paths relative to FILE.  The checkpoint is looked up as
`homography_CNN_synthetic.py --mode test` looks it up: in <--model_dir>/<--loss_type>_normalize, the `checkpoint` state
file, else the newest <--model_name>-<step>.  Without a checkpoint the run stops with an error, unless --seeded_weights
True asks for the seeded initial weights (--seed).  Files are decoded on the GPU (baseline JPEG, 8-bit PNG)
with cv2.imread for the rest.  Writes out_dir/homographies.txt (`img1 img2` and H's nine entries, row-major, '%.9g' of
their float32 values) and, with --save_warped, out_dir/<k>_warped.jpg: image 1 warped by H as written into image 2's
size, JPEG quality 95, byte-identical to cv2.imencode of cv2.warpPerspective.  Prints one line per pair and each batch's
GPU time per pair (CUDA events around prep, forward and warp).

--refine_levels N (N > 0, or -1 for levels down to a 320 px long side; default 0: off) refines each H with coarse-to-fine
ECC on the images' own pixels (align.HomographyEstimator.refine, with --refine_iters, --refine_eps, --refine_max_side):
homographies.txt and the warped files then hold the refined H, out_dir/refine.txt holds `img1 img2 rho status levels`
per pair (status 0, or the ECC failure that stopped the pair; levels: how many succeeded), and the timing line a refine term.
"""
from __future__ import absolute_import, division, print_function

import argparse
import os
import sys

import numpy as np

import homography_CNN_synthetic as syn

def build_parser():
    p = argparse.ArgumentParser(description="Homography between image pairs with a trained model")
    p.add_argument('--pairs', type=str, default=None, help='file of "img1 img2" lines, paths relative to the file')
    p.add_argument('--img1', type=str, default=None)
    p.add_argument('--img2', type=str, default=None)
    add_model_options(p)
    p.add_argument('--out_dir', type=str, default='aligned')
    p.add_argument('--save_warped', type=syn.str2bool, default='True')
    add_weights_and_refine_options(p)
    return p


def add_model_options(p):
    """The model's options, shared with mosaic_images.py: checkpoint lookup, network size, numeric mode, batch size."""
    p.add_argument('--model_dir', type=str, default=syn.MODEL_DIR)
    p.add_argument('--model_name', type=str, default='model.ckpt')
    p.add_argument('--loss_type', type=str, default='l1_loss', help='the loss the model was trained with (its subdirectory)',
                   choices=['h_loss', 'rec_loss', 'ssim_loss', 'l1_loss', 'l1_smooth_loss', 'ncc_loss'])
    p.add_argument('--img_h', type=int, default=syn.HEIGHT)
    p.add_argument('--img_w', type=int, default=syn.WIDTH)
    p.add_argument('--patch_size', type=int, default=syn.PATCH_SIZE)
    p.add_argument('--numeric', type=str, default='bf16x3', choices=['fp32', 'bf16', 'bf16x3'])
    p.add_argument('--batch_size', type=int, default=128)


def add_weights_and_refine_options(p):
    """The seeded-weights fallback and the refinement options, shared with mosaic_images.py."""
    p.add_argument('--seeded_weights', type=syn.str2bool, default='False',
                   help='without a checkpoint, use the seeded initial weights instead of stopping with an error')
    p.add_argument('--seed', type=int, default=0, help='seed of the initial weights (--seeded_weights True)')
    p.add_argument('--refine_levels', type=int, default=0,
                   help='refine H with coarse-to-fine ECC on this many levels (0: off; -1: halve down to a 320 px long side)')
    p.add_argument('--refine_iters', type=int, default=50, help='ECC iterations per refinement level')
    p.add_argument('--refine_eps', type=float, default=1e-6, help='ECC stops a level when rho changes by less than this')
    p.add_argument('--refine_max_side', type=int, default=None,
                   help='refine on images scaled to this long side at most (default: the images\' own size)')


def pair_list(args):
    """-> (names [(img1, img2)] as given, paths [(path1, path2)])."""
    from unsuperviseddeephomographyral2018_b200 import align
    if args.pairs:
        if args.img1 or args.img2:
            raise SystemExit("give --pairs or --img1/--img2, not both")
        return align.read_pairs(args.pairs)
    if not (args.img1 and args.img2):
        raise SystemExit("give --pairs FILE or both --img1 and --img2")
    return [(args.img1, args.img2)], [(args.img1, args.img2)]


def checkpoint_dir(args):
    """homography_CNN_synthetic.resolve_paths' model directory: <model_dir>/<loss_type>_normalize."""
    return os.path.join(args.model_dir, args.loss_type + "_normalize")


def make_estimator(args):
    from unsuperviseddeephomographyral2018_b200 import align
    ck, kind = syn.latest_checkpoint(checkpoint_dir(args), args.model_name)
    if not ck and not args.seeded_weights:
        raise SystemExit("no checkpoint under %s (give --model_dir / --loss_type, or --seeded_weights True for the seeded "
                         "initial weights)" % checkpoint_dir(args))
    est = align.HomographyEstimator(img_h=args.img_h, img_w=args.img_w, patch_size=args.patch_size, numeric=args.numeric,
                                    batch_size=args.batch_size, seed=args.seed)
    if ck:
        syn.restore(est.engine, ck, kind)
        print("===> model", ck)
    else:
        print("===> no checkpoint under %s: using the seeded initial weights (seed %d)" % (checkpoint_dir(args), args.seed))
    return est


def run(args, est, decode, encode):
    """Align every pair of `args`: est has estimate / warp / last_ms (align.HomographyEstimator), decode(paths) -> images
    [h,w,3] RGB, encode(images BGR [n,h,w,3]) -> JPEG bytes.  Returns the float32 homographies as written."""
    from unsuperviseddeephomographyral2018_b200 import align
    names, paths = pair_list(args)
    os.makedirs(args.out_dir, exist_ok=True)
    lines, written, refine_lines = [], np.empty((len(names), 9), np.float32), []
    refining = args.refine_levels != 0
    for c0 in range(0, len(names), args.batch_size):
        chunk = range(c0, min(c0 + args.batch_size, len(names)))
        imgs = decode([p for k in chunk for p in paths[k]])
        I1, I2 = imgs[0::2], imgs[1::2]
        H, _, _ = est.estimate(I1, I2)
        ms = dict(est.last_ms)
        if refining:
            H, rho, status, level = est.refine(I1, I2, H, None if args.refine_levels < 0 else args.refine_levels, args.refine_iters,
                                               args.refine_eps, args.refine_max_side)
            ms["refine"] = est.last_ms["refine"]
        ms["warp"] = 0.0
        n = len(chunk)
        written[c0:c0 + n] = align.homography_as_written(H)
        for j, k in enumerate(chunk):
            lines.append(align.format_line(names[k][0], names[k][1], H[j]))
            print("%s %s  H = %s" % (names[k][0], names[k][1], " ".join("%.6g" % v for v in written[k])))
            if refining:
                refine_lines.append("%s %s %.9g %d %d" % (names[k][0], names[k][1], rho[j], status[j], level[j]))
        if args.save_warped:
            import torch
            groups = {}
            for j in range(n):
                groups.setdefault((tuple(I1[j].shape), tuple(I2[j].shape[:2])), []).append(j)
            for (_, size2), js in groups.items():
                Hw = written[[c0 + j for j in js]].astype(np.float64).reshape(-1, 3, 3)
                warped = est.warp(torch.stack([I1[j] for j in js]), Hw, size2)
                ms["warp"] += est.last_ms["warp"]
                for j, blob in zip(js, encode(warped.flip(-1))):            # RGB -> cv2's BGR for the encoder
                    with open(os.path.join(args.out_dir, "%d_warped.jpg" % (c0 + j)), "wb") as f:
                        f.write(blob)
        print("===> batch of %d pairs: GPU %.3f ms/pair (prep %.3f, forward %.3f, %swarp %.3f)"
              % (n, sum(ms.values()) / n, ms["prep"] / n, ms["forward"] / n,
                 "refine %.3f, " % (ms["refine"] / n) if refining else "", ms["warp"] / n), flush=True)
    with open(os.path.join(args.out_dir, "homographies.txt"), "w") as f:
        f.write("".join(ln + "\n" for ln in lines))
    if refining:
        with open(os.path.join(args.out_dir, "refine.txt"), "w") as f:
            f.write("".join(ln + "\n" for ln in refine_lines))
    return written


def main(argv=None):
    args = build_parser().parse_args(argv)
    import torch
    from unsuperviseddeephomographyral2018_b200 import align, ops
    torch.cuda.set_device(0)
    run(args, make_estimator(args), align.decode_images, ops.encode_jpeg)
    return 0


if __name__ == "__main__":
    sys.exit(main())
