"""The mosaic's block exposure compensation (udh_mosaic_exposure_block_stats_u8, udh_exposure_block_solve and
ops.mosaic_exposure_gain_maps; the compensated blends, udh_mosaic_blend_u8 and udh_mosaic_multiband_u8 with maps):
cv2.detail_BlocksGainCompensator and cv2.detail_BlocksChannelsCompensator fed the multi-band blend's inputs, as
oracle/exposure.fed gives them (test infrastructure only).

restate() states cv2's rule in NumPy:
  blocks   per fed image (cols x rows): bpx = ceil(cols / bl_w), bw = ceil(cols / bpx), likewise bpy, bh in y.  Block
           (bx, by) is [bx bw, min(bx bw + bw, cols)) x [by bh, min(by bh + bh, rows)) of the image and its mask, its corner
           tl + (bx bw, by bh).  Blocks are numbered image-major, then row-major.
  gains    the blocks are fed, as separate images, to a GainCompensator / ChannelsCompensator with nr_feeds feeds: exactly
           oracle/exposure.restate over the blocks (a pair whose rectangles intersect but whose masks do not still adds
           beta N = beta to the diagonal and to b; a block without a positive-count pair with another block is skipped
           and gets 1).  Blocks of one image never intersect each other.
  maps     per image a bpy x bpx map of float32(gain) (3 channels in channels mode), filtered twice by
           sepFilter2D(CV_32F, [1/4, 1/2, 1/4], [1/4, 1/2, 1/4]) with BORDER_REFLECT_101: each pass is the row pass then
           the column pass, each output (a + c) 1/4 + b 1/2 in float32.  These are getMatGains()'s maps, bit for bit.
  apply    the map is resized to the image (INTER_LINEAR, float32; merged to 3 channels in gain mode) and
           v' = saturate_u8(rint(float32(v) g)) in float32 (cv2.multiply(uint8, float32 map, CV_8U)).
The resize is stated in the generic form (resize_map): per axis fx = float32((d + 0.5) (1 / (N / n)) - 0.5), s = floor(fx),
fx -= s, clamped to the border with fx = 0; a row pass S[s] (1 - fx) + S[s + 1] fx, then the column pass, each product and
sum rounded to float32.  cv2's default path (IPP, SIMD dispatch) rounds some of these values differently by 1 ulp, so the
applied bytes agree with cv2's except where float32(v) g lies within a few ulp of a rounding tie (near_tie()).
The compensated blends (feather(), multiband()): oracle/exposure.py's with apply_map in place of the per-frame gain; the
gain at a canvas pixel is the map's resize at its ROI coordinates (x - x_lo, y - y_lo).
"""
import numpy as np

from . import exposure as EX
from . import mosaic as OM
from . import multiband as MB


def grid(rows, cols, bl_w, bl_h):
    """-> (bpx, bpy, bw, bh): cv2.detail.BlocksCompensator's blocks of a rows x cols image."""
    bpx, bpy = -(-int(cols) // int(bl_w)), -(-int(rows) // int(bl_h))
    return bpx, bpy, -(-int(cols) // bpx), -(-int(rows) // bpy)


def blocks(imgs, masks, tls, bl_w, bl_h):
    """-> (block images, block masks, block corners, grids [per image (bpx, bpy, bw, bh)]) in cv2's order."""
    bi, bm, bt, grids = [], [], [], []
    for img, m, (x, y) in zip(imgs, masks, tls):
        rows, cols = m.shape[:2]
        bpx, bpy, bw, bh = g = grid(rows, cols, bl_w, bl_h)
        grids.append(g)
        for by in range(bpy):
            for bx in range(bpx):
                x0, y0 = bx * bw, by * bh
                x1, y1 = min(x0 + bw, cols), min(y0 + bh, rows)
                bi.append(np.ascontiguousarray(img[y0:y1, x0:x1]))
                bm.append(np.ascontiguousarray(m[y0:y1, x0:x1]))
                bt.append((int(x) + x0, int(y) + y0))
    return bi, bm, bt, grids


def reflect101(i, n):
    return np.where(i < 0, -i, np.where(i >= n, 2 * n - 2 - i, i)) if n > 1 else np.zeros_like(i)


def filter_pass(mp):
    """One sepFilter2D([1/4, 1/2, 1/4] both ways, BORDER_REFLECT_101) in float32: the row pass, then the column pass."""
    q, h = np.float32(0.25), np.float32(0.5)
    a = np.asarray(mp, np.float32)
    for ax in (1, 0):
        n = a.shape[ax]
        i = np.arange(n)
        lo, hi = np.take(a, reflect101(i - 1, n), ax), np.take(a, reflect101(i + 1, n), ax)
        a = (lo + hi) * q + a * h
    return a


def gain_maps(gains, grids, mode):
    """Block gains float64 [m,3] (cv2's order) -> per image its filtered map float32 [bpy,bpx] (gain) or [bpy,bpx,3]."""
    out, o = [], 0
    for bpx, bpy, _, _ in grids:
        g = np.asarray(gains[o:o + bpx * bpy], np.float64).astype(np.float32).reshape(bpy, bpx, 3)
        o += bpx * bpy
        mp = g[..., 0] if mode == "gain" else g
        for _ in range(2):
            mp = filter_pass(mp)
        out.append(mp)
    return out


def restate(imgs, masks, tls, mode="gain", feeds=1, block=32, summation="rows"):
    """Fed images, masks and top-lefts -> (maps [per image], block gains float64 [m,3], grids, per-feed block pair
    statistics): the rule above.  summation as oracle/exposure.pair_stats ("rows": cv2's row-order norm sums)."""
    bi, bm, bt, grids = blocks(imgs, masks, tls, block, block)
    g, trace = EX.restate(bi, bm, bt, mode, feeds, summation)
    return gain_maps(g, grids, mode), g, grids, trace


def _axis(n, N):
    """The generic INTER_LINEAR coefficients of an n -> N axis: (s0, s1, a0, a1) per output, float32 weights."""
    scale = 1.0 / (float(N) / float(n))
    f = ((np.arange(N) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    lo, hi = s < 0, s >= n - 1
    f[lo | hi] = 0
    s = np.clip(s, 0, n - 1)
    return s, np.minimum(s + 1, n - 1), (np.float32(1) - f).astype(np.float32), f


def resize_map(mp, rows, cols):
    """A gain map float32 [h,w] or [h,w,C] -> [rows,cols(,C)]: the generic float32 INTER_LINEAR stated above (the map itself
    when it already has the image's size, as cv2's apply does)."""
    mp = np.asarray(mp, np.float32)
    if mp.shape[:2] == (rows, cols):
        return mp
    sx0, sx1, ax0, ax1 = _axis(mp.shape[1], cols)
    sy0, sy1, ay0, ay1 = _axis(mp.shape[0], rows)
    wx = (cols,) + (1,) * (mp.ndim - 2)
    wy = (rows, 1) + (1,) * (mp.ndim - 2)
    h = mp[:, sx0] * ax0.reshape(wx) + mp[:, sx1] * ax1.reshape(wx)
    return h[sy0] * ay0.reshape(wy) + h[sy1] * ay1.reshape(wy)


def apply_map(img, mp):
    """uint8 [h,w,3] image, its (unresized) map -> saturate_u8(rint(float32(v) g)) in float32."""
    g = resize_map(mp, img.shape[0], img.shape[1])
    g = g[..., None] if g.ndim == 2 else g
    return np.clip(np.rint(np.asarray(img).astype(np.float32) * g), 0, 255).astype(np.uint8)


def near_tie(img, mp, dg):
    """bool [h,w,3]: where float32(v) g of apply_map lies within 255 dg + 2 ulp of a rounding tie (k + 1/2), so a gain
    off by at most dg can round it the other way."""
    g = resize_map(mp, img.shape[0], img.shape[1])
    g = g[..., None] if g.ndim == 2 else g
    p = np.asarray(img).astype(np.float32) * g
    return np.abs(p - (np.floor(p) + np.float32(0.5))) <= 255 * dg + 2 * np.spacing(np.abs(p) + np.float32(1))


def resize_gap(mp, rows, cols):
    """max |cv2.resize(mp) - resize_map(mp)|: how far cv2's default-path resize lies from the stated one."""
    import cv2
    a = cv2.resize(np.asarray(mp, np.float32), (int(cols), int(rows)), interpolation=cv2.INTER_LINEAR)
    return float(np.abs(a.astype(np.float64) - resize_map(mp, rows, cols).reshape(a.shape)).max())


# ---- cv2 --------------------------------------------------------------------------------------------------------------------
def cv2_maps(imgs, masks, tls, mode="gain", feeds=1, block=32):
    """cv2's block compensator fed (imgs, masks, tls) -> (maps [getMatGains(), float32], apply'd images [per image])."""
    import cv2
    cv2.ocl.setUseOpenCL(False)
    cls = cv2.detail_BlocksGainCompensator if mode == "gain" else cv2.detail_BlocksChannelsCompensator
    c = cls(int(block), int(block), int(feeds))
    tl = [(int(x), int(y)) for x, y in tls]
    c.feed(tl, [np.ascontiguousarray(i) for i in imgs], [np.ascontiguousarray(m) for m in masks])
    maps = [np.asarray(g, np.float32) for g in c.getMatGains()]
    out = [np.asarray(c.apply(k, tl[k], np.ascontiguousarray(img).copy(), masks[k])) for k, img in enumerate(imgs)]
    return maps, out


def maps(frames, M, Hc, Wc, mode="gain", feeds=1, block=32):
    """Frames, M (frame k -> canvas) -> per frame the restated map (None for a frame that is not fed)."""
    take, imgs, masks, tls = EX.fed(frames, M, Hc, Wc)
    out = [None] * len(frames)
    if take:
        for k, mp in zip(take, restate(imgs, masks, tls, mode, feeds, block)[0]):
            out[k] = mp
    return out


# ---- the compensated blends -------------------------------------------------------------------------------------------------
def feather(frames, M, Hc, Wc, feather_px, gmaps, blend_masks=None):
    """oracle/mosaic.blend with frame k's canvas warp value v replaced by saturate_u8(rint(float32(v) g)), g its resized map
    at the pixel's ROI coordinates; blend_masks (per fed frame, on its ROI) keep frame k only where set, as oracle/seam."""
    import cv2
    from unsuperviseddeephomographyral2018_b200 import mosaic
    M = np.asarray(M, np.float64).reshape(-1, 3, 3)
    rois, _ = mosaic.multiband_rois(M, [f.shape[:2] for f in frames], Hc, Wc)
    take = [k for k in range(len(frames)) if rois[k, 2] > rois[k, 0] and rois[k, 3] > rois[k, 1]]
    C = frames[0].shape[2] if frames[0].ndim == 3 else 1
    S = np.zeros((Hc, Wc, C), np.int64)
    D = np.zeros((Hc, Wc), np.int64)
    for k in take:
        F, Mk = frames[k], M[k]
        h, w = F.shape[:2]
        x0, y0, x1, y1 = (int(v) for v in rois[k])
        v = cv2.warpPerspective(F if C == 3 else F.reshape(h, w), Mk, (Wc, Hc)).reshape(Hc, Wc, C)
        _, wt = OM.validity_weight(Mk, h, w, Hc, Wc, feather_px)
        g = np.ones((Hc, Wc, 3), np.float32)
        r = resize_map(gmaps[k], y1 - y0, x1 - x0)
        g[y0:y1, x0:x1] = r[..., None] if r.ndim == 2 else r
        v = np.clip(np.rint(v.astype(np.float32) * g[..., :C]), 0, 255).astype(np.int64)
        on = np.zeros((Hc, Wc), bool)
        on[y0:y1, x0:x1] = True
        if blend_masks is not None:
            on[y0:y1, x0:x1] = blend_masks[take.index(k)] != 0
        wt = np.where(on, wt, 0)
        S += wt[..., None] * v
        D += wt
    out = np.where(D[..., None] > 0, (S + (D >> 1)[..., None]) // np.maximum(D, 1)[..., None], 0).astype(np.uint8)
    return out, np.where(D > 0, 255, 0).astype(np.uint8)


def multiband(frames, M, Hc, Wc, bands, gmaps, blend_masks=None):
    """oracle/multiband.cv2_blend fed apply_map(img_k, gmaps[k]) for each fed frame k, with its blend mask (per fed frame)
    in place of its validity mask when given."""
    take, imgs, masks, tls = EX.fed(frames, M, Hc, Wc)
    imgs = [apply_map(img, gmaps[k]) for img, k in zip(imgs, take)]
    out, mask, _ = MB.cv2_blend(imgs, masks if blend_masks is None else blend_masks, tls, Hc, Wc, bands)
    return out, mask
