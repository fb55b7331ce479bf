"""The mosaic's seams (udh_mosaic_seam_masks_u8, bit for bit): cv2.detail's Voronoi seam finder fed the multi-band blend's
inputs, and the blend masks it leaves (test infrastructure only).

Inputs: exactly what oracle/multiband.fed gives the blender, for each fed frame k (those whose ROI meets the canvas, in
index order): its validity mask mask_k uint8 [roi_h,roi_w] (255 where the ROI warp is valid, else 0) and its ROI's
top-left tl_k = (x, y).  cv2_seams() calls cv2.detail.SeamFinder_createDefault(SeamFinder_VORONOI_SEAM).find with OpenCL
off; restate() states its rule in NumPy:
  pairs      (0, 1), (0, 2), .., (0, n-1), (1, 2), ..: every pair i < j whose ROI rectangles intersect, in that order; each
             pair reads the masks as the pairs before it left them, so the order is part of the result.
  window     the ROIs' intersection grown by GAP = 10 px on every side (not clipped); s_i = frame i's mask where the window
             pixel lies inside frame i's ROI, 0 elsewhere (likewise s_j).
  unique     u_i = s_i and not s_j, u_j = s_j and not s_i.
  distances  d_i = the exact L1 distance from each window pixel to the nearest u_i pixel of the window (cv2's DIST_L1, mask
             3); +inf (cv2: FLT_MAX) everywhere when the window holds no u_i pixel.  Computed here as two separable
             passes: the distance along the column, then min over x' of g(x') + |x - x'| by a prefix and a suffix minimum.
  assignment over the intersection only: where d_i < d_j frame j's mask is cleared, elsewhere frame i's (ties and two
             infinite distances clear frame i).  So a frame whose window holds none of its own unique pixels is cleared
             from the whole intersection, and a frame lying inside another one vanishes: that is cv2's result, kept.
blend_masks(): what cv2's stitcher then feeds the blender, cv2.dilate(seam_k, None) (3 x 3 rectangle, a border that never
wins) AND mask_k.  The end-to-end references feed those masks to oracle/multiband.cv2_blend (optionally with the images
compensated first, the order of cv2's stitcher: its compensator sees the un-seamed masks) and to the feathered blend, where
frame k contributes at a canvas pixel only where it is valid by oracle/mosaic.py's rule and its blend mask is set.
"""
import numpy as np

from . import exposure as EX
from . import mosaic as OM
from . import multiband as MB

GAP = 10
INF = np.iinfo(np.int64).max // 4


def cv2_seams(masks, tls):
    """Fed masks (uint8 [h,w]) and top-lefts -> the seam masks cv2's Voronoi finder leaves (uint8 [h,w] each)."""
    import cv2
    cv2.ocl.setUseOpenCL(False)
    finder = cv2.detail.SeamFinder_createDefault(cv2.detail.SeamFinder_VORONOI_SEAM)
    imgs = [np.zeros(m.shape + (3,), np.float32) for m in masks]
    out = finder.find(imgs, [(int(x), int(y)) for x, y in tls], [cv2.UMat(np.ascontiguousarray(m)) for m in masks])
    return [np.asarray(u.get() if isinstance(u, cv2.UMat) else u, np.uint8) for u in out]


def pairs(tls, shapes):
    """[(i, j, (x0, y0, x1, y1))]: the pairs i < j whose ROIs intersect, in cv2's visiting order."""
    r = [(x, y, x + s[1], y + s[0]) for (x, y), s in zip(tls, shapes)]
    return [(i, j, rect) for i, j, rect in EX.pairs(r) if i != j]


def l1_distance(src):
    """bool [h,w] -> int64 [h,w]: the exact L1 distance to the nearest True pixel (INF where there is none)."""
    h, w = src.shape
    y = np.arange(h)[:, None]
    last = np.maximum.accumulate(np.where(src, y, -INF), 0)                        # nearest source at or above
    nxt = np.minimum.accumulate(np.where(src, y, INF)[::-1], 0)[::-1]               # ... at or below
    g = np.minimum(np.where(last > -INF, y - last, INF), np.where(nxt < INF, nxt - y, INF))
    x = np.arange(w)[None, :]
    pre = np.minimum.accumulate(np.where(g < INF, g - x, INF), 1)                    # min over x' <= x of g(x') - x'
    suf = np.minimum.accumulate(np.where(g < INF, g + x, INF)[:, ::-1], 1)[:, ::-1]  # min over x' >= x of g(x') + x'
    d = np.minimum(np.where(pre < INF, pre + x, INF), np.where(suf < INF, suf - x, INF))
    return np.where(d >= INF // 2, INF, d)


def _window(m, tl, x0, y0, x1, y1):
    """Frame mask m at top-left tl on the window (x0 - GAP, y0 - GAP) .. (x1 + GAP, y1 + GAP): bool, False outside it."""
    out = np.zeros((y1 - y0 + 2 * GAP, x1 - x0 + 2 * GAP), bool)
    h, w = m.shape
    ax, ay = x0 - GAP - tl[0], y0 - GAP - tl[1]                                      # window origin in frame coordinates
    sx0, sy0, sx1, sy1 = max(ax, 0), max(ay, 0), min(ax + out.shape[1], w), min(ay + out.shape[0], h)
    if sx0 < sx1 and sy0 < sy1:
        out[sy0 - ay:sy1 - ay, sx0 - ax:sx1 - ax] = m[sy0:sy1, sx0:sx1] != 0
    return out


def find_in_pair(mi, mj, tli, tlj, rect, tie_to_j=True):
    """One pair's step, in place on mi and mj (uint8 masks); rect is the ROIs' intersection (x0, y0, x1, y1)."""
    x0, y0, x1, y1 = rect
    si, sj = _window(mi, tli, *rect), _window(mj, tlj, *rect)
    both = si & sj
    di, dj = l1_distance(si & ~both), l1_distance(sj & ~both)
    inner = (slice(GAP, GAP + y1 - y0), slice(GAP, GAP + x1 - x0))
    keep_i = di[inner] < dj[inner] if tie_to_j else di[inner] <= dj[inner]
    vi = mi[y0 - tli[1]:y1 - tli[1], x0 - tli[0]:x1 - tli[0]]
    vj = mj[y0 - tlj[1]:y1 - tlj[1], x0 - tlj[0]:x1 - tlj[0]]
    vj[keep_i] = 0
    vi[~keep_i] = 0


def restate(masks, tls):
    """Fed masks and top-lefts -> the seam masks (uint8 [h,w] each): the rule above in NumPy."""
    out = [np.array(m, np.uint8, copy=True) for m in masks]
    for i, j, rect in pairs(tls, [m.shape for m in out]):
        find_in_pair(out[i], out[j], tls[i], tls[j], rect)
    return out


def blend_masks(seams, masks):
    """-> cv2.dilate(seam_k, None) AND mask_k per frame: the masks cv2's stitcher feeds its blender."""
    import cv2
    return [cv2.bitwise_and(cv2.dilate(s, None), m) for s, m in zip(seams, masks)]


def fed(frames, M, Hc, Wc):
    """-> (take, imgs, masks, tls) as oracle/multiband.fed feeds the blender (oracle/exposure.fed)."""
    return EX.fed(frames, M, Hc, Wc)


def multiband(frames, M, Hc, Wc, bands, gains=None):
    """cv2's seams of the fed masks -> blend masks -> oracle/multiband.cv2_blend, fed apply(img_k, gains[k]) with gains
    -> (mosaic uint8 [Hc,Wc,3], mask uint8 [Hc,Wc])."""
    take, imgs, masks, tls = fed(frames, M, Hc, Wc)
    if gains is not None:
        g = np.asarray(gains, np.float64).reshape(len(frames), -1)
        imgs = [EX.apply(img, np.broadcast_to(g[k], (3,))) for img, k in zip(imgs, take)]
    bm = blend_masks(cv2_seams(masks, tls), masks)
    out, mask, _ = MB.cv2_blend(imgs, bm, tls, Hc, Wc, bands)
    return out, mask


def feather(frames, M, Hc, Wc, feather_px, gains=None):
    """oracle/mosaic.blend (oracle/exposure.feather with gains) with frame k's weight kept only where its blend mask from
    cv2's seams is set; a frame that is not fed contributes nothing."""
    import cv2
    take, _, masks, tls = fed(frames, M, Hc, Wc)
    bm = blend_masks(cv2_seams(masks, tls), masks)
    on = [np.zeros((Hc, Wc), bool) for _ in frames]
    for k, b, (x, y) in zip(take, bm, tls):
        on[k][y:y + b.shape[0], x:x + b.shape[1]] = b != 0
    C = frames[0].shape[2] if frames[0].ndim == 3 else 1
    g = np.ones((len(frames), 3)) if gains is None else np.asarray(gains, np.float64).reshape(len(frames), -1)
    S = np.zeros((Hc, Wc, C), np.int64)
    D = np.zeros((Hc, Wc), np.int64)
    for k, (F, Mk) in enumerate(zip(frames, np.asarray(M, np.float64).reshape(-1, 3, 3))):
        h, w = F.shape[:2]
        v = cv2.warpPerspective(F if C == 3 else F.reshape(h, w), Mk, (Wc, Hc)).reshape(Hc, Wc, C)
        if gains is not None:
            v = EX.apply(v, g[k][:C] if len(g[k]) >= C else g[k][0])
        _, wt = OM.validity_weight(Mk, h, w, Hc, Wc, feather_px)
        wt = np.where(on[k], wt, 0)
        S += wt[..., None] * v.astype(np.int64)
        D += wt
    out = np.where(D[..., None] > 0, (S + (D >> 1)[..., None]) // np.maximum(D, 1)[..., None], 0).astype(np.uint8)
    return out, np.where(D > 0, 255, 0).astype(np.uint8)
