"""Stitch an image sequence into one mosaic: chain the learned pairwise homographies to a reference frame, lay out a
canvas, and blend every frame onto it on the GPU (udh_mosaic_blend_u8, or udh_mosaic_multiband_u8 across frequency bands).

    out = build_mosaic(est, frames, ref=None, refine=None, feather=64, max_pixels=None, blend="feather", bands=5,
                       compensate="none", compensate_feeds=1, seam="none", seam_megapix=None)
    out["mosaic"], out["mask"], out["M"], out["kept"], out["H_pairs"], out["gains"], out["last_ms"]

frames are CUDA uint8 RGB [h_k,w_k,3] tensors in sequence order (sizes may differ); est is an align.HomographyEstimator.

Chaining.  H_k maps frame k to frame k + 1 (align's image 1 -> image 2).  chain_to_reference gives G_k, frame k -> the
reference frame: G_ref = I, G_k = n(G_{k+1} H_k) below the reference and G_k = n(G_{k-1} inv(H_{k-1})) above it, with n
normalising [2,2] to 1.  The default reference is the middle frame N // 2, which halves the longest chain.  Errors of the
pairwise H's accumulate along the chain (drift); nothing here closes loops or adjusts the chain globally.

Canvas.  canvas() drops a frame (never the reference) when a corner of its source rectangle grown by 1 px, (-1, -1) ..
(w, h), maps with a denominator <= 0: such a frame reaches the line at infinity.  Over the kept frames' mapped pixel-centre
corners (0, 0), (w - 1, 0), (w - 1, h - 1), (0, h - 1): x0 = floor(min x), Wc = ceil(max x) - x0 + 1, likewise in y, and
M_k = T G_k with T the translation by (-x0, -y0).

Blend, blend="feather" (the default).  oracle/mosaic.py states the rule: per canvas pixel, the integer feathered average of
every frame's cv2.warpPerspective(F_k, M_k, (Wc, Hc)) value where the frame is valid, with weights 1 + min(distance to the
frame's edge in 1/32 px, 32 feather).

Blend, blend="multiband".  oracle/multiband.py states the rule: cv2.detail_MultiBandBlender(0, bands, CV_16S) (Burt-Adelson:
low frequencies blended over a wide region, high ones over a narrow one), fed each frame's warp on its ROI
(multiband_rois) with the feathered blend's validity as its mask.  It hides the seams a drifting chain leaves where a
feathered average would ghost.  An exposure step between frames it only spreads over its low-frequency region; exposure
compensation removes it.

Exposure compensation, compensate="gain" or "channels" (default "none").  Before either blend, ops.mosaic_exposure_gains
computes what cv2.detail_GainCompensator(compensate_feeds) (one gain per frame) or ChannelsCompensator (one per channel)
finds for the kept frames' ROI warps (oracle/exposure.py states the rule); the blend then takes each frame's warp value
as saturate_u8(rint(v g)).  This is the stage cv2's stitcher runs between the warp and the blender.  compensate=
"gain_blocks" or "channels_blocks" runs cv2's default, the block compensators (oracle/exposure_blocks.py): a gain per
block of about compensate_block px of each ROI warp, whose filtered map ops.mosaic_exposure_gain_maps returns and the
blend applies per pixel, so brightness that varies across a frame (vignetting) is compensated too.

Seams, seam="voronoi" (default "none").  ops.mosaic_seam_masks cuts the kept frames' validity masks apart as
cv2.detail's Voronoi seam finder does (oracle/seam.py states the rule): pair by pair in cv2's order, each pixel of an
overlap goes to the frame whose own pixels lie nearer in L1 distance.  Each frame then blends only where the 3 x 3
dilation of its seam mask meets its validity (cv2's stitcher's blend mask): the multi-band blend switches the high
frequencies at the seam and spreads only the low ones, instead of averaging the frames across the whole overlap, which
leaves a semi-transparent double image where the chain drifts; the feathered blend keeps its weights inside each
frame's region.  The compensator still sees the un-seamed masks, as in cv2's stitcher.  A frame lying inside another
one's region gets nothing (cv2's result).  seam="gc_color" cuts each overlap as cv2.detail's GraphCutSeamFinder
(COST_COLOR) does instead (oracle/seam_gc.py): along the minimum cut of a graph whose edges cost the two warps' squared
colour difference, so the seam runs where the frames agree rather than where geometry puts it.

Seam scale, seam_megapix=m (default None: full resolution).  As cv2's stitcher (stitching_detailed's --seam_megapix,
Stitcher::setSeamEstimationResol), the seams are found on the frames scaled by a = min(1, sqrt(m 1e6 / area of frame 0))
(seam_scale; oracle/seam_scale.py states the rule): each frame resized by a with INTER_LINEAR_EXACT, the finder on the
pixel-centre conjugates C(a) M_k C(a)^-1 over a ceil(a Hc) x ceil(a Wc) seam canvas (seam_geometry), and each frame's
dilated seam mask sampled back at its full-resolution canvas positions, AND its validity: graded blend masks.  The
multi-band blend weighs a frame mask + 1 there (cv2's feed), the feathered one keeps it where the mask is nonzero.  The
finder's cost falls with a^2: the graph-cut finder becomes usable on camera-size sweeps.  The seam-scale frames cover up
to about 1 / (2a) px less at each edge, so a few valid pixels at the mosaic's outer border can get no weight (mask 0
there, as in cv2).  a = 1 is the full-resolution path.
"""
import math

import numpy as np

MAX_SIDE = 32766                 # udh_mosaic_blend_u8 takes canvas sides below 32767


def _normalise(G):
    return G / G[2, 2]


def chain_to_reference(H_pairs, ref=None):
    """H_pairs [N-1,3,3] (frame k -> frame k + 1) -> (G float64 [N,3,3] frame k -> frame ref with G[k][2,2] = 1, ref)."""
    H = np.asarray(H_pairs, np.float64).reshape(-1, 3, 3)
    N = len(H) + 1
    ref = N // 2 if ref is None or ref < 0 else int(ref)
    if ref >= N:
        raise ValueError("reference frame %d of a %d-frame sequence" % (ref, N))
    G = np.empty((N, 3, 3))
    G[ref] = np.eye(3)
    for k in range(ref - 1, -1, -1):
        G[k] = _normalise(G[k + 1] @ H[k])
    for k in range(ref + 1, N):
        G[k] = _normalise(G[k - 1] @ np.linalg.inv(H[k - 1]))
    return G, ref


def _map(G, pts):
    p = np.asarray(pts, np.float64) @ np.asarray(G, np.float64).T
    return p[:, 0] / p[:, 2], p[:, 1] / p[:, 2], p[:, 2]


def grown_corners(h, w):
    return np.array([[-1.0, -1.0, 1.0], [w, -1.0, 1.0], [w, h, 1.0], [-1.0, h, 1.0]])


def centre_corners(h, w):
    return np.array([[0.0, 0.0, 1.0], [w - 1.0, 0.0, 1.0], [w - 1.0, h - 1.0, 1.0], [0.0, h - 1.0, 1.0]])


def canvas(sizes, G, ref, max_pixels=None):
    """sizes [(h_k, w_k)], G [N,3,3] (frame k -> reference) -> (M float64 [N,3,3] frame k -> canvas, (Hc, Wc), kept bool
    [N]).  ValueError naming the frame with the corner farthest from the reference frame's centre when a side exceeds
    MAX_SIDE or, with max_pixels, Hc Wc > max_pixels."""
    G = np.asarray(G, np.float64).reshape(-1, 3, 3)
    kept = np.ones(len(G), bool)
    xs, ys = [], []
    for k, (h, w) in enumerate(sizes):
        with np.errstate(all="ignore"):
            _, _, den = _map(G[k], grown_corners(h, w))
            x, y, _ = _map(G[k], centre_corners(h, w))
        if k != ref and not ((den > 0).all() and np.isfinite(x).all() and np.isfinite(y).all()):
            kept[k] = False
            continue
        xs.append(x); ys.append(y)
    xs, ys = np.concatenate(xs), np.concatenate(ys)
    x0, y0 = np.floor(xs.min()), np.floor(ys.min())
    Wc, Hc = int(np.ceil(xs.max()) - x0) + 1, int(np.ceil(ys.max()) - y0) + 1
    if max(Hc, Wc) > MAX_SIDE or (max_pixels is not None and Hc * Wc > max_pixels):
        raise ValueError("the %dx%d canvas exceeds %s; frame %d reaches farthest from the reference frame (drop it or pick "
                         "another --ref_frame)" % (Hc, Wc, "%d px a side" % MAX_SIDE if max(Hc, Wc) > MAX_SIDE else
                                                   "%d pixels" % max_pixels, farthest_frame(sizes, G, kept, ref)))
    T = np.array([[1.0, 0.0, -x0], [0.0, 1.0, -y0], [0.0, 0.0, 1.0]])
    return T @ G, (Hc, Wc), kept


def multiband_rois(M, sizes, Hc, Wc):
    """M [n,3,3] (frame k -> canvas), sizes [(h_k, w_k)] -> (rois int64 [n,4] (x_lo, y_lo, x_hi, y_hi), M' float64 [n,3,3]
    frame k -> its ROI): the canvas rectangle the multi-band blend warps frame k onto.  Over the mapped pixel-centre corners,
    x_lo = max(0, floor(min x) - 1), x_hi = min(Wc, ceil(max x) + 2) (exclusive), likewise in y; M'_k = T(-x_lo, -y_lo) M_k.
    The margin holds every pixel whose warp is valid (its source position rounds to within 1/64 px of the frame).  An ROI
    that misses the canvas is empty (x_hi <= x_lo or y_hi <= y_lo).  ValueError for a frame whose grown corners map with a
    denominator <= 0 or whose corners do not map to finite points: canvas() drops such frames."""
    M = np.asarray(M, np.float64).reshape(-1, 3, 3)
    rois = np.zeros((len(M), 4), np.int64)
    Mr = np.empty_like(M)
    for k, (h, w) in enumerate(sizes):
        with np.errstate(all="ignore"):
            _, _, den = _map(M[k], grown_corners(h, w))
            x, y, _ = _map(M[k], centre_corners(h, w))
        if not ((den > 0).all() and np.isfinite(x).all() and np.isfinite(y).all()):
            raise ValueError("frame %d: its corners do not map to finite points in front of the canvas's camera" % k)
        x0, y0 = max(0, int(np.floor(x.min())) - 1), max(0, int(np.floor(y.min())) - 1)
        x1, y1 = min(int(Wc), int(np.ceil(x.max())) + 2), min(int(Hc), int(np.ceil(y.max())) + 2)
        rois[k] = (x0, y0, x1, y1)
        Mr[k] = np.array([[1.0, 0.0, -x0], [0.0, 1.0, -y0], [0.0, 0.0, 1.0]]) @ M[k]
    return rois, Mr


def farthest_frame(sizes, G, kept, ref):
    """The kept frame whose mapped pixel-centre corner lies farthest from the reference frame's centre."""
    h, w = sizes[ref]
    cx, cy = (w - 1) / 2.0, (h - 1) / 2.0
    best, far = -1.0, ref
    for k, (h, w) in enumerate(sizes):
        if kept[k]:
            x, y, _ = _map(G[k], centre_corners(h, w))
            d = np.hypot(x - cx, y - cy).max()
            if d > best:
                best, far = d, k
    return far


def seam_scale(sizes, megapix):
    """cv2's seam scale: a = min(1, sqrt(megapix 1e6 / (h0 w0))) of the first frame's size (h0, w0)."""
    h0, w0 = sizes[0]
    if not megapix > 0:
        raise ValueError("seam_megapix must be > 0 (got %r)" % (megapix,))
    return min(1.0, math.sqrt(float(megapix) * 1e6 / (float(h0) * float(w0))))


def centre_map(a):
    """C(a): a pixel centre -> the centre it maps to in an image resized by a (cv2.resize's own sampling map)."""
    return np.array([[a, 0.0, a / 2.0 - 0.5], [0.0, a, a / 2.0 - 0.5], [0.0, 0.0, 1.0]])


def seam_geometry(M, sizes, Hc, Wc, a):
    """M [n,3,3] (frame k -> canvas), sizes [(h_k, w_k)] -> (M^s [n,3,3] = C(a) M_k C(a)^-1, the resized frames' sizes
    [(rint(a h_k), rint(a w_k))], the seam canvas (ceil(a Hc), ceil(a Wc))).  ValueError for a frame resized to nothing."""
    C = centre_map(a)
    Ci = np.linalg.inv(C)
    Ms = np.stack([C @ Mk @ Ci for Mk in np.asarray(M, np.float64).reshape(-1, 3, 3)])
    small = [(int(np.rint(h * a)), int(np.rint(w * a))) for h, w in sizes]
    for k, (h, w) in enumerate(small):
        if h < 1 or w < 1:
            raise ValueError("frame %d (%dx%d) is empty at seam scale %.17g" % (k, sizes[k][0], sizes[k][1], a))
    return Ms, small, (int(math.ceil(a * Hc)), int(math.ceil(a * Wc)))


COMPENSATE = ("none", "gain", "channels", "gain_blocks", "channels_blocks")
SEAM = ("none", "voronoi", "gc_color")


def build_mosaic(est, frames, ref=None, refine=None, feather=64, max_pixels=None, float32_M=False, blend="feather", bands=5,
                 compensate="none", compensate_feeds=1, seam="none", compensate_block=32, seam_megapix=None):
    """est: align.HomographyEstimator; frames: CUDA uint8 RGB [h_k,w_k,3] tensors in sequence order.  blend: "feather"
    (udh_mosaic_blend_u8 with `feather`) or "multiband" (udh_mosaic_multiband_u8 with `bands`).  refine: None, or a
    dict of est.refine's keyword arguments (levels, iters, eps, max_side) to refine each pair's H.  max_pixels: the canvas
    limit (None: the JPEG encoder's, udh_jpeg_encode_capacity(Hc, Wc, 3) != 0).  float32_M: blend with each M_k rounded to
    float32, the values a text file of '%.9g' float32 entries gives back.  compensate: "none", "gain" or "channels"
    (ops.mosaic_exposure_gains with compensate_feeds feeds, applied by the blend), or "gain_blocks" / "channels_blocks"
    (ops.mosaic_exposure_gain_maps with blocks of about compensate_block px: a gain map per frame, cv2's
    BlocksGainCompensator / BlocksChannelsCompensator; gains stay 1).  seam: "none", "voronoi" or "gc_color"
    (ops.mosaic_seam_masks' finder; each frame blends only inside its blend mask).  seam_megapix: None (full resolution)
    or m > 0, the seams found at seam_scale(sizes, m) (a seam is needed).
    -> dict(mosaic uint8 [Hc,Wc,3] RGB, mask uint8 [Hc,Wc], M [N,3,3] frame k -> canvas (float64, float32 values with
    float32_M), kept bool [N], ref, H_pairs [N-1,3,3], refine (rho, status, level_reached) or None, gains float64 [N,3]
    (1 for a dropped frame, all 1 without per-frame compensation), gain_maps [N] (the block modes only: CUDA float32
    maps, None for a dropped frame or one whose ROI misses the canvas), seam_scale (a; 1 at full resolution), last_ms {prep,
    forward, refine, compensate, seam, blend} of CUDA-event time; compensate only when compensating, seam only with seams,
    covering the resize, the finder and the upscale at a seam scale)."""
    frames = list(frames)
    if len(frames) < 2:
        raise ValueError("a mosaic needs at least two frames (got %d)" % len(frames))
    H, _, _ = est.estimate(frames[:-1], frames[1:])
    ms = dict(est.last_ms)
    refined = None
    if refine is not None:
        H, rho, status, reached = est.refine(frames[:-1], frames[1:], H, **refine)
        refined = (rho, status, reached)
        ms["refine"] = est.last_ms["refine"]
    G, ref = chain_to_reference(H, ref)
    sizes = [tuple(int(v) for v in f.shape[:2]) for f in frames]
    M, (Hc, Wc), kept = canvas(sizes, G, ref, max_pixels)
    if float32_M:
        M = M.astype(np.float32).astype(np.float64)
    if max_pixels is None:
        check_encodable(Hc, Wc, sizes, G, kept, ref)
    if blend not in ("feather", "multiband"):
        raise ValueError("blend must be 'feather' or 'multiband' (got %r)" % (blend,))
    if compensate not in COMPENSATE:
        raise ValueError("compensate must be one of %s (got %r)" % (", ".join(COMPENSATE), compensate))
    if seam not in SEAM:
        raise ValueError("seam must be one of %s (got %r)" % (", ".join(SEAM), seam))
    if seam_megapix is not None and seam == "none":
        raise ValueError("seam_megapix needs a seam finder")
    a = 1.0 if seam_megapix is None else seam_scale(sizes, seam_megapix)
    gains = np.ones((len(frames), 3))
    gain_maps = None
    if compensate in ("gain", "channels"):
        gains[kept], ms["compensate"] = compensate_kept(frames, M, kept, Hc, Wc, compensate, compensate_feeds)
    elif compensate != "none":
        gain_maps, ms["compensate"] = compensate_blocks_kept(frames, M, kept, Hc, Wc, compensate[:-len("_blocks")], compensate_feeds,
                                                             compensate_block)
    masks = None
    if seam != "none":
        masks, ms["seam"] = seam_kept(frames, M, kept, Hc, Wc, seam, a)
    mosaic, mask, ms["blend"] = blend_kept(frames, M, kept, Hc, Wc, feather, blend, bands,
                                           gains if compensate in ("gain", "channels") else None, masks,
                                           None if gain_maps is None else [gain_maps[k] for k in range(len(frames)) if kept[k]])
    out = dict(mosaic=mosaic, mask=mask, M=M, kept=kept, ref=ref, H_pairs=H, refine=refined, gains=gains, seam_scale=a, last_ms=ms)
    if gain_maps is not None:
        out["gain_maps"] = gain_maps
    return out


def check_encodable(Hc, Wc, sizes, G, kept, ref):
    """ValueError unless the JPEG encoder takes an Hc x Wc colour image, naming the frame that reaches farthest."""
    from . import _lib
    if _lib.lib.udh_jpeg_encode_capacity(Hc, Wc, 3) == 0:
        raise ValueError("the %dx%d canvas is larger than the JPEG encoder takes; frame %d reaches farthest from the reference "
                         "frame (drop it or pick another --ref_frame)" % (Hc, Wc, farthest_frame(sizes, G, kept, ref)))


def compensate_kept(frames, M, kept, Hc, Wc, mode, feeds=1):
    """The kept frames' exposure gains (ops.mosaic_exposure_gains) -> (gains float64 [n_kept,3], CUDA-event ms)."""
    import torch
    from . import ops
    take = [k for k in range(len(frames)) if kept[k]]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g = ops.mosaic_exposure_gains([frames[k].contiguous() for k in take], np.asarray(M)[take], Hc, Wc, mode, feeds)
    e1.record()
    e1.synchronize()
    return g, e0.elapsed_time(e1)


def compensate_blocks_kept(frames, M, kept, Hc, Wc, mode, feeds=1, block=32):
    """The kept frames' block gain maps (ops.mosaic_exposure_gain_maps) -> (maps [N], None for a dropped frame or one whose
    ROI misses the canvas; CUDA-event ms)."""
    import torch
    from . import ops
    take = [k for k in range(len(frames)) if kept[k]]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g = ops.mosaic_exposure_gain_maps([frames[k].contiguous() for k in take], np.asarray(M)[take], Hc, Wc, mode, feeds, block)
    e1.record()
    e1.synchronize()
    maps = [None] * len(frames)
    for q, k in enumerate(take):
        maps[k] = g[q]
    return maps, e0.elapsed_time(e1)


def seam_kept(frames, M, kept, Hc, Wc, finder="voronoi", scale=1.0):
    """The kept frames' blend masks (ops.mosaic_seam_masks with finder at scale) -> (masks [n_kept]: CUDA uint8 [roi_h,roi_w],
    None for a frame whose ROI misses the canvas; CUDA-event ms)."""
    import torch
    from . import ops
    take = [k for k in range(len(frames)) if kept[k]]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    s = ops.mosaic_seam_masks([frames[k].contiguous() for k in take], np.asarray(M)[take], Hc, Wc, finder, scale)
    e1.record()
    e1.synchronize()
    masks = [None] * len(take)
    for q, b in zip(s["take"], s["blend"]):
        masks[q] = b
    return masks, e0.elapsed_time(e1)


def blend_kept(frames, M, kept, Hc, Wc, feather, mode="feather", bands=5, gains=None, masks=None, gain_maps=None):
    """The kept frames through ops.mosaic_blend_u8 (mode "feather") or ops.mosaic_multiband_u8 ("multiband") -> (mosaic,
    mask, CUDA-event ms).  gains: None, or [N,3] per frame (exposure compensation).  masks: None, or seam_kept's blend
    masks of the kept frames.  gain_maps: None, or the kept frames' block gain maps."""
    import torch
    from . import ops
    take = [k for k in range(len(frames)) if kept[k]]
    g = None if gains is None else np.asarray(gains, np.float64)[take]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    if mode == "multiband":
        mosaic, mask = ops.mosaic_multiband_u8([frames[k].contiguous() for k in take], np.asarray(M)[take], Hc, Wc, bands,
                                               gains=g, masks=masks, gain_maps=gain_maps)
    else:
        mosaic, mask = ops.mosaic_blend_u8([frames[k].contiguous() for k in take], np.asarray(M)[take], Hc, Wc, feather,
                                           gains=g, masks=masks, gain_maps=gain_maps)
    e1.record()
    e1.synchronize()
    return mosaic, mask, e0.elapsed_time(e1)
