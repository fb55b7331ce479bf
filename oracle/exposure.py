"""The mosaic's exposure compensation (udh_mosaic_exposure_stats_u8 and ops.mosaic_exposure_gains; the compensated blends,
udh_mosaic_blend_u8 and udh_mosaic_multiband_u8 with gains): cv2.detail_GainCompensator and cv2.detail_ChannelsCompensator
fed the multi-band blend's inputs (test infrastructure only).

Inputs: exactly what oracle/multiband.fed gives the blender, for each kept frame k whose ROI meets the canvas: corner_k =
tl_k, img_k = cv2.warpPerspective(F_k, M'_k, roi size), mask_k = 255 where the pixel is valid.  A frame whose ROI misses the
canvas is not fed and gets gain 1.

restate() states cv2's rule in NumPy:
  statistics  for every pair i <= j (i = j included) whose ROI rectangles intersect: c = the pixels of the intersection
              where both masks are set; N_ij = N_ji = max(1, c) (0 for rectangles that do not intersect).  Where c > 0:
              I_ij = sum s_i / N_ij, I_ji = sum s_j / N_ij, and for i != j neither frame is skipped.  Mode "gain": s =
              sqrt(double(r^2 + g^2 + b^2)) (cv2's norm(Vec3b)), summed by cv2 in row order; mode "channels": s is one
              channel's value and every channel is compensated on its own.
  system      over the unskipped frames in index order, alpha = 0.01, beta = 100, for j ascending: b_i += beta N_ij,
              A_ii += beta N_ij and, if j != i, A_ii += 2 alpha I_ij^2 N_ij, A_ij -= 2 alpha I_ij I_ji N_ij; gains =
              cv2.solve(A, b) (DECOMP_LU); skipped frames get 1.
  feeds       with F feeds, feed t sees every image apply'd with the gains of feeds 0..t-1 in turn (each apply rounds to
              uint8); the gains are the element-wise product of the feeds'.
  apply       v' = saturate_u8(rint(v g)) in float64, ties to even (cv2.multiply(uint8, double)).
The compensated blends: feather() is oracle/mosaic.py with each frame's warp value apply'd before it is weighted;
multiband() is oracle/multiband.py fed apply'd ROI warps, the order of cv2's stitcher.
"""
import math

import numpy as np

from . import mosaic as OM
from . import multiband as MB

ALPHA, BETA = 0.01, 100.0


def apply(img, g):
    """uint8 [..., C] image, gain (scalar or [C]) -> saturate_u8(rint(img g)) in float64."""
    return np.clip(np.rint(np.asarray(img).astype(np.float64) * np.asarray(g, np.float64)), 0, 255).astype(np.uint8)


# ---- cv2 --------------------------------------------------------------------------------------------------------------------
def compensator(mode, feeds):
    import cv2
    return cv2.detail_GainCompensator(int(feeds)) if mode == "gain" else cv2.detail_ChannelsCompensator(int(feeds))


def cv2_gains(imgs, masks, tls, mode="gain", feeds=1):
    """Fed images, masks and top-lefts -> (gains float64 [m,3] (gain mode: one gain repeated), the fed compensator)."""
    c = compensator(mode, feeds)
    c.feed([(int(x), int(y)) for x, y in tls], [np.ascontiguousarray(i) for i in imgs], list(masks))
    g = np.array([np.asarray(v, np.float64).reshape(-1)[:3 if mode == "channels" else 1] for v in c.getMatGains()]).reshape(len(imgs), -1)
    return np.ascontiguousarray(np.broadcast_to(g, (len(imgs), 3))), c


def fed(frames, M, Hc, Wc):
    """-> (take: the indices of the fed frames, imgs, masks, tls) as oracle/multiband.fed feeds the blender."""
    from unsuperviseddeephomographyral2018_b200 import mosaic
    M = np.asarray(M, np.float64).reshape(-1, 3, 3)
    rois, _ = mosaic.multiband_rois(M, [f.shape[:2] for f in frames], Hc, Wc)
    take = [k for k in range(len(frames)) if rois[k, 2] > rois[k, 0] and rois[k, 3] > rois[k, 1]]
    imgs, masks, tls = MB.fed(frames, M, Hc, Wc)
    return take, imgs, masks, tls


def gains(frames, M, Hc, Wc, mode="gain", feeds=1):
    """Kept frames uint8 RGB [h_k,w_k,3], M [n,3,3] (frame k -> canvas) -> float64 [n,3]: cv2's compensator on the multi-band
    inputs (1 for a frame that is not fed)."""
    take, imgs, masks, tls = fed(frames, M, Hc, Wc)
    out = np.ones((len(frames), 3), np.float64)
    if take:
        out[take] = cv2_gains(imgs, masks, tls, mode, feeds)[0]
    return out


# ---- the restatement --------------------------------------------------------------------------------------------------------
def pairs(rois):
    """[(i, j, (x0, y0, x1, y1))] of the pairs i <= j whose rectangles (x_lo, y_lo, x_hi, y_hi) intersect."""
    out = []
    for i in range(len(rois)):
        for j in range(i, len(rois)):
            x0, y0 = max(rois[i][0], rois[j][0]), max(rois[i][1], rois[j][1])
            x1, y1 = min(rois[i][2], rois[j][2]), min(rois[i][3], rois[j][3])
            if x0 < x1 and y0 < y1:
                out.append((i, j, (x0, y0, x1, y1)))
    return out


def norms(img):
    """uint8 [..., 3] -> cv2's norm(Vec3b) per pixel: sqrt(double(r^2 + g^2 + b^2))."""
    return np.sqrt(np.sum(np.asarray(img).astype(np.int64) ** 2, -1).astype(np.float64))


def pair_stats(imgs, masks, tls, summation="exact"):
    """-> list of dict(i, j, count, sums int64 [2,3] (frame i's and j's channel sums), norms float64 [2]) per intersecting
    pair i <= j.  summation: "exact" (math.fsum: the exact sum, rounded once) or "rows" (cv2's running sum in row order)."""
    rois = [(x, y, x + m.shape[1], y + m.shape[0]) for (x, y), m in zip(tls, masks)]
    out = []
    for i, j, (x0, y0, x1, y1) in pairs(rois):
        si = (slice(y0 - tls[i][1], y1 - tls[i][1]), slice(x0 - tls[i][0], x1 - tls[i][0]))
        sj = (slice(y0 - tls[j][1], y1 - tls[j][1]), slice(x0 - tls[j][0], x1 - tls[j][0]))
        both = (masks[i][si] == 255) & (masks[j][sj] == 255)
        vi, vj = imgs[i][si][both], imgs[j][sj][both]                  # row-major order
        if summation == "exact":
            ns = [math.fsum(norms(vi)), math.fsum(norms(vj))]
        else:
            ns = [float(np.add.accumulate(norms(v))[-1]) if len(v) else 0.0 for v in (vi, vj)]
        out.append(dict(i=i, j=j, count=int(both.sum()), sums=np.stack([vi.astype(np.int64).sum(0), vj.astype(np.int64).sum(0)]),
                        norms=np.array(ns)))
    return out


def solve(m, stats, isum):
    """One feed's gains [m] from pair statistics; isum(p) -> (sum s_i, sum s_j) of pair p."""
    import cv2
    N = np.zeros((m, m), np.int64)
    I = np.zeros((m, m))
    skip = np.ones(m, bool)
    for p in stats:
        i, j = p["i"], p["j"]
        N[i, j] = N[j, i] = max(1, p["count"])
        if p["count"] == 0:
            continue
        if i != j:
            skip[i] = skip[j] = False
        s1, s2 = isum(p)
        I[i, j], I[j, i] = float(s1) / N[i, j], float(s2) / N[i, j]
    g = np.ones(m)
    keep = np.flatnonzero(~skip)
    if not len(keep):
        return g
    A = np.zeros((len(keep), len(keep)))
    b = np.zeros((len(keep), 1))
    for ki, i in enumerate(keep):
        for kj, j in enumerate(keep):
            b[ki, 0] += BETA * int(N[i, j])
            A[ki, ki] += BETA * int(N[i, j])
            if j != i:
                A[ki, ki] += 2 * ALPHA * float(I[i, j]) * float(I[i, j]) * int(N[i, j])
                A[ki, kj] -= 2 * ALPHA * float(I[i, j]) * float(I[j, i]) * int(N[i, j])
    g[keep] = cv2.solve(A, b)[1].reshape(-1)
    return g


def restate(imgs, masks, tls, mode="gain", feeds=1, summation="exact"):
    """Fed images, masks and top-lefts -> (gains float64 [m,3], [per feed: its pair_stats]): the rule above in NumPy."""
    m = len(imgs)
    cur = [np.asarray(i) for i in imgs]
    acc, trace = None, []
    for _ in range(int(feeds)):
        st = pair_stats(cur, masks, tls, summation)
        trace.append(st)
        if mode == "gain":
            g3 = np.repeat(solve(m, st, lambda p: p["norms"])[:, None], 3, 1)
        else:
            g3 = np.stack([solve(m, st, lambda p, c=c: p["sums"][:, c]) for c in range(3)], 1)
        acc = g3.copy() if acc is None else acc * g3
        cur = [apply(img, g) for img, g in zip(cur, g3)]
    return acc, trace


# ---- the compensated blends -------------------------------------------------------------------------------------------------
def feather(frames, M, Hc, Wc, feather_px, gains):
    """oracle/mosaic.blend with each frame's warp value v replaced by apply(v, gains[k]) before it is weighted."""
    import cv2
    C = frames[0].shape[2] if frames[0].ndim == 3 else 1
    S = np.zeros((Hc, Wc, C), np.int64)
    D = np.zeros((Hc, Wc), np.int64)
    for F, Mk, g in zip(frames, np.asarray(M, np.float64).reshape(-1, 3, 3), np.asarray(gains, np.float64).reshape(len(frames), -1)):
        h, w = F.shape[:2]
        v = cv2.warpPerspective(F if C == 3 else F.reshape(h, w), Mk, (Wc, Hc)).reshape(Hc, Wc, C)
        v = apply(v, g[:C] if len(g) >= C else g[0]).astype(np.int64)
        _, wt = OM.validity_weight(Mk, h, w, Hc, Wc, feather_px)
        S += wt[..., None] * v
        D += wt
    out = np.where(D[..., None] > 0, (S + (D >> 1)[..., None]) // np.maximum(D, 1)[..., None], 0).astype(np.uint8)
    return out, np.where(D > 0, 255, 0).astype(np.uint8)


def multiband(frames, M, Hc, Wc, bands, gains):
    """oracle/multiband.blend fed apply(img_k, gains[k]) for each fed frame k."""
    take, imgs, masks, tls = fed(frames, M, Hc, Wc)
    g = np.asarray(gains, np.float64).reshape(len(frames), -1)
    imgs = [apply(img, np.broadcast_to(g[k], (3,))) for img, k in zip(imgs, take)]
    out, mask, _ = MB.cv2_blend(imgs, masks, tls, Hc, Wc, bands)
    return out, mask
