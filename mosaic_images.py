#!/usr/bin/env python
"""Stitch an image sequence into one mosaic with a trained model: the homography of every consecutive pair (frame k ->
frame k + 1, as align_images.py computes it), chained to a reference frame, and every frame blended onto one canvas on the
GPU (unsuperviseddeephomographyral2018_b200.mosaic states the chaining, the canvas and the blend rule).

    python mosaic_images.py --frames raw/ --model_dir ../models/real_models/ --img_h 142 --img_w 190
    python mosaic_images.py --frames frames.txt --seeded_weights True --refine_levels -1 --out_dir mosaic/

--frames takes a list file (one path per line, relative to the file, in sequence order) or a directory, read as
sorted(glob(dir/--glob)) (default *.JPG, gen_real_data.py's rule).  The model, refinement and batch options are
align_images.py's.  --ref_frame picks the reference frame (-1: the middle one, N // 2); --feather is the blend's ramp in
source pixels (0: a plain average of the overlapping frames).  --blend multiband blends across --bands frequency bands
instead (cv2.detail_MultiBandBlender's rule, byte for byte): low frequencies over a wide region, high ones over a narrow
one, which hides the seams a drifting chain leaves.  --compensate gain|channels compensates each frame's exposure before
the blend (cv2.detail_GainCompensator / ChannelsCompensator's rule with --compensate_feeds feeds): one gain per frame, or
one per channel, which also evens out white balance.  --compensate gain_blocks|channels_blocks (cv2's stitcher's default,
cv2.detail_BlocksGainCompensator / BlocksChannelsCompensator) solves for a gain per block of about --compensate_block px
of each frame and applies the smoothed map of them, which also removes brightness that varies across a frame, such as
vignetting.  An exposure step between frames is otherwise left in the mosaic.
cv2's rule pulls every gain towards 1, so one feed removes only part of a step; each further feed removes part of what
is left (on a sweep with exposures 0.75 / 1 / 1.3, four gain-mode feeds recover the gain ratios to within 1 %).
--seam voronoi cuts seams between the frames before the blend (cv2.detail's Voronoi seam finder, byte for byte): each
pixel of an overlap goes to one frame, so the blend no longer averages two drifted frames into a double image across
the whole overlap; with --blend multiband only the low frequencies are spread across the seam.  --seam gc_color cuts
them as cv2.detail's GraphCutSeamFinder(COST_COLOR) does, as the exact minimum cut of each overlap's colour-difference
graph: the seam runs where the two frames agree.  --seam_megapix X finds the seams at a reduced resolution, as cv2's
stitcher does (its default is 0.1): the frames scaled to about X megapixels (by the first frame's area) with
INTER_LINEAR_EXACT, the seams found there, and each seam mask resampled back to full resolution (graded along the seam).
The graph-cut finder's time falls with the pixel count; -1 (the default) keeps full resolution.

Writes in --out_dir:
  pairs.txt    `frame_k frame_k+1` and H's nine entries per consecutive pair, as align_images.py's homographies.txt;
  refine.txt   with refinement, `frame_k frame_k+1 rho status levels` per pair, as align_images.py writes it;
  mosaic.txt   `canvas Hc Wc ref r` (` blend multiband B` appended with --blend multiband, then ` compensate MODE F` with
               --compensate, then ` seam <finder>` with --seam, ` seam <finder> A` when --seam_megapix gives a seam
               scale A < 1, '%.17g'), then `name kept|dropped` and the nine entries of M_k (frame k -> canvas) per frame,
               '%.9g' of their float32 values; the blend uses those float32 values.  With --compensate each frame line
               ends in its three gains, '%.17g' (exact); so the file reproduces mosaic.jpg.  With a block mode the
               compensate field is ` compensate MODE F B` (B: --compensate_block) and the frame lines carry no gains;
  gain_maps.npz with --compensate gain_blocks|channels_blocks, each fed frame's gain map (float32 [bpy,bpx] or
               [bpy,bpx,3], keyed by frame name), as cv2's compensator's getMatGains() returns it;
  mosaic.jpg   the mosaic (BGR, JPEG quality 95, byte-identical to cv2.imencode of the same pixels).
A frame whose grown corners map behind the reference camera is dropped.  The canvas must be one the JPEG encoder takes
(about 110 MP in colour); a larger one stops with an error naming the frame that reaches farthest.  Prints the GPU time
of each phase (CUDA events: prep, forward, refine, compensate, seam, blend, encode; the blend named when it is
multi-band).
"""
from __future__ import absolute_import, division, print_function

import argparse
import glob
import os
import sys

import numpy as np

import align_images


def build_parser():
    p = argparse.ArgumentParser(description="Stitch an image sequence into one mosaic with a trained model")
    p.add_argument('--frames', type=str, required=True, help='list file (one path per line, relative to it) or directory')
    p.add_argument('--glob', type=str, default='*.JPG', help='the frames of a --frames directory: sorted(glob(dir/GLOB))')
    align_images.add_model_options(p)
    align_images.add_weights_and_refine_options(p)
    p.add_argument('--ref_frame', type=int, default=-1, help='reference frame (-1: the middle one)')
    p.add_argument('--feather', type=int, default=64, help='blend ramp in source pixels, 0..1024 (0: plain average)')
    p.add_argument('--blend', type=str, default='feather', choices=['feather', 'multiband'],
                   help='feather: feathered average; multiband: blend across frequency bands')
    p.add_argument('--bands', type=int, default=5, help='frequency bands of --blend multiband, 0..10')
    p.add_argument('--compensate', type=str, default='none', choices=['none', 'gain', 'channels', 'gain_blocks', 'channels_blocks'],
                   help='exposure compensation before the blend: none, one gain per frame, one per channel, or a smooth '
                        'map of gains per block of each frame (gain_blocks: one gain, channels_blocks: one per channel)')
    p.add_argument('--compensate_block', type=int, default=32,
                   help='block side in pixels of --compensate gain_blocks|channels_blocks, 1..1024')
    p.add_argument('--compensate_feeds', type=int, default=1,
                   help='feeds of the exposure compensator, 1..16; one feed removes only part of an exposure step (the '
                        'rule pulls every gain towards 1), several (e.g. 4) remove nearly all of it')
    p.add_argument('--seam', type=str, default='none', choices=['none', 'voronoi', 'gc_color'],
                   help='seams between the frames before the blend: none, cv2.detail\'s Voronoi seam finder, or its '
                        'GraphCutSeamFinder(COST_COLOR) as an exact minimum cut')
    p.add_argument('--seam_megapix', type=float, default=-1,
                   help='find the seams on frames scaled to about this many megapixels (cv2\'s seam_megapix; needs --seam); '
                        '-1: at full resolution')
    p.add_argument('--out_dir', type=str, default='mosaic')
    return p


def frame_list(args):
    """-> (names as written in mosaic.txt, paths) in sequence order."""
    if os.path.isdir(args.frames):
        paths = sorted(glob.glob(os.path.join(args.frames, args.glob)))
        names = [os.path.basename(p) for p in paths]
    else:
        base = os.path.dirname(os.path.abspath(args.frames))
        with open(args.frames) as f:
            names = [ln.strip() for ln in f if ln.strip()]
        paths = [os.path.join(base, nm) for nm in names]
    if len(paths) < 2:
        raise SystemExit("%s: a mosaic needs at least two frames (found %d)" % (args.frames, len(paths)))
    return names, paths


def run(args, est, decode, encode):
    """Mosaic the frames of `args`: est is an align.HomographyEstimator, decode(paths) -> CUDA RGB images, encode(images
    BGR [n,h,w,3]) -> JPEG bytes.  Returns build_mosaic's result."""
    import torch
    from unsuperviseddeephomographyral2018_b200 import align, mosaic
    if not 0 <= args.feather <= 1024:
        raise SystemExit("--feather must be in 0..1024 (got %d)" % args.feather)
    if not 0 <= args.bands <= 10:
        raise SystemExit("--bands must be in 0..10 (got %d)" % args.bands)
    if not 1 <= args.compensate_feeds <= 16:
        raise SystemExit("--compensate_feeds must be in 1..16 (got %d)" % args.compensate_feeds)
    if not 1 <= args.compensate_block <= 1024:
        raise SystemExit("--compensate_block must be in 1..1024 (got %d)" % args.compensate_block)
    if args.seam_megapix > 0 and args.seam == "none":
        raise SystemExit("--seam_megapix needs --seam")
    names, paths = frame_list(args)
    os.makedirs(args.out_dir, exist_ok=True)
    refining = args.refine_levels != 0
    refine = dict(levels=None if args.refine_levels < 0 else args.refine_levels, iters=args.refine_iters, eps=args.refine_eps,
                  max_side=args.refine_max_side) if refining else None
    compensating = args.compensate != "none"
    blocks = args.compensate.endswith("_blocks")
    comp = dict(compensate=args.compensate, compensate_feeds=args.compensate_feeds) if compensating else {}
    if blocks:
        comp["compensate_block"] = args.compensate_block
    seaming = args.seam != "none"
    if seaming:
        comp["seam"] = args.seam
        if args.seam_megapix > 0:
            comp["seam_megapix"] = args.seam_megapix
    imgs = decode(paths)
    try:
        out = mosaic.build_mosaic(est, imgs, None if args.ref_frame < 0 else args.ref_frame, refine, args.feather,
                                  float32_M=True, blend=args.blend, bands=args.bands, **comp)
    except ValueError as e:
        raise SystemExit(str(e))
    H = out["H_pairs"]
    with open(os.path.join(args.out_dir, "pairs.txt"), "w") as f:
        f.write("".join(align.format_line(names[k], names[k + 1], H[k]) + "\n" for k in range(len(H))))
    if refining:
        rho, status, level = out["refine"]
        with open(os.path.join(args.out_dir, "refine.txt"), "w") as f:
            f.write("".join("%s %s %.9g %d %d\n" % (names[k], names[k + 1], rho[k], status[k], level[k]) for k in range(len(H))))
    Hc, Wc = out["mask"].shape
    lines = ["canvas %d %d ref %d" % (Hc, Wc, out["ref"]) + (" blend multiband %d" % args.bands if args.blend == "multiband" else "") +
             (" compensate %s %d" % (args.compensate, args.compensate_feeds) if compensating else "") +
             (" %d" % args.compensate_block if blocks else "") +
             (" seam %s" % args.seam if seaming else "") +
             (" %.17g" % out["seam_scale"] if seaming and out.get("seam_scale", 1.0) < 1.0 else "")]
    for k, nm in enumerate(names):
        lines.append(" ".join([nm, "kept" if out["kept"][k] else "dropped"] +
                              ["%.9g" % v for v in align.homography_as_written(out["M"][k])[0]] +
                              (["%.17g" % g for g in out["gains"][k]] if compensating and not blocks else [])))
        if not out["kept"][k]:
            print("===> dropped %s: it maps behind the reference frame's camera" % nm)
    with open(os.path.join(args.out_dir, "mosaic.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
    if blocks:
        np.savez(os.path.join(args.out_dir, "gain_maps.npz"),
                 **{nm: m.cpu().numpy() for nm, m in zip(names, out["gain_maps"]) if m is not None})
    ms = out["last_ms"]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    blob = encode(out["mosaic"].flip(-1)[None])[0]                       # RGB -> cv2's BGR for the encoder
    e1.record()
    e1.synchronize()
    ms["encode"] = e0.elapsed_time(e1)
    with open(os.path.join(args.out_dir, "mosaic.jpg"), "wb") as f:
        f.write(blob)
    cover = float((out["mask"] != 0).float().mean())
    print("===> %d frames (%d kept) on a %dx%d canvas (ref %s, %.1f %% covered): GPU %.3f ms (prep %.3f, forward %.3f, %s%s"
          "%s%sblend %.3f, encode %.3f)" % (len(names), int(np.sum(out["kept"])), Hc, Wc, names[out["ref"]], 100 * cover,
                                            sum(ms.values()), ms["prep"], ms["forward"],
                                            "refine %.3f, " % ms["refine"] if refining else "",
                                            "compensate %.3f, " % ms["compensate"] if compensating else "",
                                            "seam %.3f, " % ms["seam"] if seaming else "",
                                            "multiband %d " % args.bands if args.blend == "multiband" else "", ms["blend"],
                                            ms["encode"]), flush=True)
    return out


def main(argv=None):
    args = build_parser().parse_args(argv)
    import torch
    from unsuperviseddeephomographyral2018_b200 import align, ops
    torch.cuda.set_device(0)
    run(args, align_images.make_estimator(args), align.decode_images, ops.encode_jpeg)
    return 0


if __name__ == "__main__":
    sys.exit(main())
