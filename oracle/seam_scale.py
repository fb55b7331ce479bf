"""Seams found at a reduced resolution (cv2's seam_megapix), as ops.mosaic_seam_masks(..., scale=a) computes them, byte for
byte (test infrastructure only).

With seam_megapix m > 0 and frame 0 of h0 x w0 (cv2 takes the first image's area, whatever the others' sizes):
  scale     a = min(1, sqrt(m 1e6 / (h0 w0))).  a == 1 is the full-resolution path, unchanged.
  frames    F^s_k = cv2.resize(F_k, None, fx=a, fy=a, interpolation=INTER_LINEAR_EXACT): the fx form, whose sampling
            scale is a itself (an explicit dsize would use dsize / size instead, and give other bytes).
  geometry  C(a) = [[a, 0, a/2 - 1/2], [0, a, a/2 - 1/2], [0, 0, 1]] maps a pixel centre to the resized image's (the
            resize's own sampling map); M^s_k = C(a) M_k C(a)^-1, the seam canvas is (ceil(a Hc), ceil(a Wc)), the seam ROIs
            are mosaic.multiband_rois(M^s, seam sizes, seam canvas), and the finder (oracle/seam or oracle/seam_gc) runs
            unchanged on (F^s, M^s, seam canvas).
  masks     frame k's blend mask at full-ROI pixel (X, Y) of the canvas: D_k = cv2.dilate(seam^s_k, None), placed on the
            seam canvas with 0 outside its seam ROI, sampled by INTER_LINEAR_EXACT arithmetic at the seam-canvas position
            ((X + 1/2) a - 1/2, (Y + 1/2) a - 1/2), AND (bytewise) the frame's full-resolution validity (0 / 255).  The
            masks are graded: 1 .. 254 along the seams.  A frame whose full ROI meets the canvas but whose seam ROI does not
            gets an all-zero mask.
  blends    the feathered blend keeps a frame where its mask is nonzero; the multi-band blend weighs it mask + 1 there
            (cv2's CV_16S feed rule, oracle/multiband.py).  The compensator still sees the full-resolution validity.

INTER_LINEAR_EXACT on uint8 (cv2.resize's bit-exact path), per axis of a source of n pixels: scale = 1 / inv_scale (inv_scale
= fx, or dsize / size), f = (d + 1/2) scale - 1/2 in float64, s = floor(f), c1 = rint((f - s) 256) (ties to even), c0 =
256 - c1, taps (s, s + 1); both taps are pixel 0 when s < 0 and pixel n - 1 when s + 1 > n - 1.  The horizontal sums h =
c0 p(s) + c1 p(s + 1) of two rows, then v = c0' h0 + c1' h1, and (v + 2^15) >> 16.  An output of the source's size is a copy
(cv2 returns the source whatever fx says).
"""
import math

import numpy as np

from . import exposure as EX
from . import exposure_blocks as EB
from . import mosaic as OM
from . import multiband as MB
from . import seam as SM
from . import seam_gc as GC


# ---- INTER_LINEAR_EXACT -----------------------------------------------------------------------------------------------
def exact_axis(n, N, scale):
    """-> (s0, s1, c1) int64 [N]: the taps and the upper weight of an n -> N axis sampled at (d + 1/2) scale - 1/2."""
    f = (np.arange(N, dtype=np.float64) + 0.5) * float(scale) - 0.5
    s = np.floor(f)
    c1 = np.rint((f - s) * 256.0).astype(np.int64)
    s = s.astype(np.int64)
    s0 = np.where(s < 0, 0, np.where(s + 1 > n - 1, n - 1, s))
    s1 = np.where(s < 0, 0, np.where(s + 1 > n - 1, n - 1, s + 1))
    return s0, s1, c1


def fx_size(n, a):
    """cv2.resize's output side for fx = a: saturate_cast<int>(n a), rounding half to even."""
    return int(np.rint(n * float(a)))


def resize_exact(img, dst_h=None, dst_w=None, fx=None, fy=None):
    """cv2.resize(img, (dst_w, dst_h)) or cv2.resize(img, None, fx=fx, fy=fy) with INTER_LINEAR_EXACT on uint8 [h,w] or
    [h,w,C], restated."""
    img = np.asarray(img, np.uint8)
    h, w = img.shape[:2]
    if fx is not None:
        fy = fx if fy is None else fy
        dst_h, dst_w, ix, iy = fx_size(h, fy), fx_size(w, fx), float(fx), float(fy)
    else:
        ix, iy = dst_w / float(w), dst_h / float(h)
    if (dst_h, dst_w) == (h, w):                                    # cv2 copies when the size stays, whatever fx says
        return img.copy()
    return sample(img.astype(np.int64), exact_axis(w, dst_w, 1.0 / ix), exact_axis(h, dst_h, 1.0 / iy)).astype(np.uint8)


def sample(src, cols, rows):
    """int64 [h,w(,C)], column taps and row taps (exact_axis) -> the INTER_LINEAR_EXACT values (int64)."""
    xs0, xs1, xc1 = cols
    ys0, ys1, yc1 = rows
    ex = (slice(None),) + (None,) * (src.ndim - 2)
    hz = lambda r: r[:, xs0] * (256 - xc1)[ex] + r[:, xs1] * xc1[ex]
    h0, h1 = hz(src[ys0]), hz(src[ys1])
    ey = (slice(None), None) + (None,) * (src.ndim - 2)
    return (h0 * (256 - yc1)[ey] + h1 * yc1[ey] + (1 << 15)) >> 16


# ---- the scale and the seam geometry -------------------------------------------------------------------------------------
def seam_scale(sizes, megapix):
    """a = min(1, sqrt(megapix 1e6 / (h0 w0))) of the first frame."""
    h0, w0 = sizes[0]
    return min(1.0, math.sqrt(float(megapix) * 1e6 / (float(h0) * float(w0))))


def centre_map(a):
    return np.array([[a, 0.0, a / 2.0 - 0.5], [0.0, a, a / 2.0 - 0.5], [0.0, 0.0, 1.0]])


def seam_geometry(M, sizes, Hc, Wc, a):
    """-> (M^s [n,3,3], seam sizes [(h, w)], (Hs, Ws))."""
    C = centre_map(a)
    Ms = np.stack([C @ Mk @ np.linalg.inv(C) for Mk in np.asarray(M, np.float64).reshape(-1, 3, 3)])
    return Ms, [(fx_size(h, a), fx_size(w, a)) for h, w in sizes], (int(math.ceil(a * Hc)), int(math.ceil(a * Wc)))


def seams(frames, M, Hc, Wc, a, finder="voronoi"):
    """-> (take_s, seam masks on the seam ROIs, seam rois int64 [n,4], M^s, (Hs, Ws)): the finder on the resized frames."""
    from unsuperviseddeephomographyral2018_b200 import mosaic
    Ms, ssizes, (Hs, Ws) = seam_geometry(M, [f.shape[:2] for f in frames], Hc, Wc, a)
    Fs = [resize_exact(f, fx=a, fy=a) for f in frames]
    take, imgs, masks, tls = SM.fed(Fs, Ms, Hs, Ws)
    found = GC.restate(imgs, masks, tls)[0] if finder == "gc_color" else SM.restate(masks, tls)
    rois, _ = mosaic.multiband_rois(Ms, ssizes, Hs, Ws)
    return take, found, rois, Ms, (Hs, Ws)


def upscale_taps(N, a, n):
    """The taps of canvas axis 0 .. N - 1 on a seam-canvas axis of n pixels: sampled at (X + 1/2) a - 1/2."""
    return exact_axis(n, N, a)


def blend_masks(frames, M, Hc, Wc, a, take_s, seams_s, rois_s, seam_canvas):
    """The full-resolution blend masks (per frame whose full ROI meets the canvas, uint8 on its ROI) of seam-scale seams
    (seams_s per frame of take_s, on rois_s)."""
    import cv2
    from unsuperviseddeephomographyral2018_b200 import mosaic
    M = np.asarray(M, np.float64).reshape(-1, 3, 3)
    rois, Mr = mosaic.multiband_rois(M, [f.shape[:2] for f in frames], Hc, Wc)
    Hs, Ws = seam_canvas
    cols, rows = upscale_taps(Wc, a, Ws), upscale_taps(Hc, a, Hs)
    out = []
    for k in range(len(frames)):
        x0, y0, x1, y1 = (int(v) for v in rois[k])
        if x1 <= x0 or y1 <= y0:
            continue
        D = np.zeros((Hs, Ws), np.int64)
        if k in take_s:
            sx0, sy0, sx1, sy1 = (int(v) for v in rois_s[k])
            D[sy0:sy1, sx0:sx1] = cv2.dilate(seams_s[take_s.index(k)], None)
        v = sample(D, tuple(t[x0:x1] for t in cols), tuple(t[y0:y1] for t in rows))
        valid, _ = OM.validity_weight(Mr[k], frames[k].shape[0], frames[k].shape[1], y1 - y0, x1 - x0, 0)
        out.append(np.where(valid, v, 0).astype(np.uint8))
    return out


def masks(frames, M, Hc, Wc, a, finder="voronoi"):
    """-> (take, blend masks [per fed frame], seam-scale seams (take_s, seams, rois_s, seam canvas)): the rule above."""
    take_s, found, rois_s, _, canvas_s = seams(frames, M, Hc, Wc, a, finder)
    take, _, _, _ = EX.fed(frames, M, Hc, Wc)
    return take, blend_masks(frames, M, Hc, Wc, a, take_s, found, rois_s, canvas_s), (take_s, found, rois_s, canvas_s)


# ---- the blends ---------------------------------------------------------------------------------------------------------------
def multiband(frames, M, Hc, Wc, bands, bm, gains=None, gmaps=None):
    """oracle/multiband.cv2_blend fed the (optionally compensated) ROI warps with the blend masks bm (per fed frame)."""
    if gmaps is not None:
        return EB.multiband(frames, M, Hc, Wc, bands, gmaps, bm)
    take, imgs, _, tls = EX.fed(frames, M, Hc, Wc)
    if gains is not None:
        g = np.asarray(gains, np.float64).reshape(len(frames), -1)
        imgs = [EX.apply(img, np.broadcast_to(g[k], (3,))) for img, k in zip(imgs, take)]
    out, mask, _ = MB.cv2_blend(imgs, bm, tls, Hc, Wc, bands)
    return out, mask


def feather(frames, M, Hc, Wc, feather_px, bm, gains=None, gmaps=None):
    """oracle/mosaic.blend (with gains, oracle/exposure's apply; with gain maps, oracle/exposure_blocks') with frame k's
    weight kept only where its blend mask (bm, per fed frame) is nonzero."""
    import cv2
    from unsuperviseddeephomographyral2018_b200 import mosaic
    if gmaps is not None:
        return EB.feather(frames, M, Hc, Wc, feather_px, gmaps, bm)
    M = np.asarray(M, np.float64).reshape(-1, 3, 3)
    rois, _ = mosaic.multiband_rois(M, [f.shape[:2] for f in frames], Hc, Wc)
    take = [k for k in range(len(frames)) if rois[k, 2] > rois[k, 0] and rois[k, 3] > rois[k, 1]]
    C = frames[0].shape[2] if frames[0].ndim == 3 else 1
    g = None if gains is None else np.asarray(gains, np.float64).reshape(len(frames), -1)
    S = np.zeros((Hc, Wc, C), np.int64)
    D = np.zeros((Hc, Wc), np.int64)
    for k in take:
        F, Mk = frames[k], M[k]
        h, w = F.shape[:2]
        x0, y0, x1, y1 = (int(v) for v in rois[k])
        v = cv2.warpPerspective(F if C == 3 else F.reshape(h, w), Mk, (Wc, Hc)).reshape(Hc, Wc, C)
        if g is not None:
            v = EX.apply(v, g[k][:C] if len(g[k]) >= C else g[k][0])
        _, wt = OM.validity_weight(Mk, h, w, Hc, Wc, feather_px)
        on = np.zeros((Hc, Wc), bool)
        on[y0:y1, x0:x1] = bm[take.index(k)] != 0
        wt = np.where(on, wt, 0)
        S += wt[..., None] * v.astype(np.int64)
        D += wt
    out = np.where(D[..., None] > 0, (S + (D >> 1)[..., None]) // np.maximum(D, 1)[..., None], 0).astype(np.uint8)
    return out, np.where(D > 0, 255, 0).astype(np.uint8)
