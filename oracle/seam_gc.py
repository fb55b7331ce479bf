"""The mosaic's graph-cut seams (udh_mosaic_seam_gc_masks_u8, bit for bit): cv2.detail's GraphCutSeamFinder(COST_COLOR)
fed the multi-band blend's inputs, as the canonical minimum cut (test infrastructure only).

Inputs: what oracle/multiband.fed gives the blender, per fed frame k: its ROI warp img_k uint8 [roi_h,roi_w,3] (border
values included), its validity mask mask_k and its ROI's top-left tl_k.  cv2_seams() calls
cv2.detail_GraphCutSeamFinder('COST_COLOR').find on float32 copies of the warps with OpenCL off; restate() states the rule:
  pairs      oracle/seam.pairs (cv2's visiting order); each pair reads the masks as the earlier pairs left them.
  window     oracle/seam's: the intersection grown by GAP on every side, s_i = frame i's mask inside its ROI, 0 outside;
             I_i = frame i's warp inside its ROI, 0 outside (likewise for j).
  graph      d(p) = sum_c (I_i(p) - I_j(p))^2; edge (p, q) between right and down neighbours, d(p) + d(q) + 1 both ways,
             + PENALTY unless s_i and s_j hold both p and q; source TERM where s_i and not s_j, sink TERM where s_j and not
             s_i (cv2's addTermWeights cancels the common TERM of a pixel both masks hold).
  cut        T = the pixels that reach the sink in the residual graph of a maximum flow (the same for every maximum flow
             and every maximum preflow), S = the rest; every capacity is an integer below 2^24, so cv2's float graph cuts
             exactly too.  Where the minimum cut is unique cv2's S is this S; where it is not, cv2's lies between the
             smallest and the largest minimum source set (bounds()).
  update     over the intersection: p in S where frame i holds it clears frame j's mask, p in T where frame j holds it
             clears frame i's (cv2's inSourceSegment branch).
Blend masks are oracle/seam.blend_masks of the result, as for the Voronoi finder.  The grid graphs use the layout of
udh_debug_grid_mincut: hcap[y,x] for edge (x, y) - (x + 1, y), vcap[y,x] for (x, y) - (x, y + 1), src and snk.
"""
import numpy as np

from . import exposure as EX
from . import seam as SM

GAP = SM.GAP
TERM = 10000
PENALTY = 1000


def cv2_seams(imgs, masks, tls):
    """Fed warps (uint8 [h,w,3]), masks and top-lefts -> the seam masks cv2's COST_COLOR graph-cut finder leaves."""
    import cv2
    cv2.ocl.setUseOpenCL(False)
    finder = cv2.detail_GraphCutSeamFinder("COST_COLOR")
    out = finder.find([np.asarray(i, np.float32) for i in imgs], [(int(x), int(y)) for x, y in tls],
                      [cv2.UMat(np.ascontiguousarray(m)) for m in masks])
    return [np.asarray(u.get() if isinstance(u, cv2.UMat) else u, np.uint8) for u in out]


def _window_img(img, tl, x0, y0, x1, y1):
    out = np.zeros((y1 - y0 + 2 * GAP, x1 - x0 + 2 * GAP, 3), np.int64)
    h, w = img.shape[:2]
    ax, ay = x0 - GAP - tl[0], y0 - GAP - tl[1]
    sx0, sy0, sx1, sy1 = max(ax, 0), max(ay, 0), min(ax + out.shape[1], w), min(ay + out.shape[0], h)
    if sx0 < sx1 and sy0 < sy1:
        out[sy0 - ay:sy1 - ay, sx0 - ax:sx1 - ax] = img[sy0:sy1, sx0:sx1]
    return out


def window_graph(Ii, Ij, si, sj):
    """Window warps (int [h,w,3]) and masks (bool [h,w]) -> (hcap, vcap, src, snk) int64 [h,w]."""
    d = ((Ii.astype(np.int64) - Ij.astype(np.int64)) ** 2).sum(-1)
    both = si & sj
    hcap, vcap = np.zeros_like(d), np.zeros_like(d)
    hcap[:, :-1] = d[:, :-1] + d[:, 1:] + 1 + np.where(both[:, :-1] & both[:, 1:], 0, PENALTY)
    vcap[:-1] = d[:-1] + d[1:] + 1 + np.where(both[:-1] & both[1:], 0, PENALTY)
    return hcap, vcap, np.where(si & ~sj, TERM, 0), np.where(sj & ~si, TERM, 0)


def pair_graph(imgs, masks, tls, i, j, rect):
    """Pair (i, j)'s window graph on the masks as they stand -> (hcap, vcap, src, snk)."""
    si, sj = SM._window(masks[i], tls[i], *rect), SM._window(masks[j], tls[j], *rect)
    return window_graph(_window_img(imgs[i], tls[i], *rect), _window_img(imgs[j], tls[j], *rect), si, sj)


def _edges(hcap, vcap, src, snk):
    """-> (u, v, c) of every directed edge with c > 0; vertex h w is the source, h w + 1 the sink."""
    h, w = hcap.shape
    idx = np.arange(h * w).reshape(h, w)
    u = [idx[:, :-1].ravel(), idx[:, 1:].ravel(), idx[:-1].ravel(), idx[1:].ravel(), np.full(h * w, h * w), idx.ravel()]
    v = [idx[:, 1:].ravel(), idx[:, :-1].ravel(), idx[1:].ravel(), idx[:-1].ravel(), idx.ravel(), np.full(h * w, h * w + 1)]
    c = [hcap[:, :-1].ravel(), hcap[:, :-1].ravel(), vcap[:-1].ravel(), vcap[:-1].ravel(), src.ravel(), snk.ravel()]
    u, v, c = np.concatenate(u), np.concatenate(v), np.concatenate(c).astype(np.int64)
    keep = c > 0
    return u[keep], v[keep], c[keep]


def _reach(n, u, v, start):
    """bool [n]: the vertices reachable from start along the directed edges u -> v."""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import breadth_first_order
    g = csr_matrix((np.ones(len(u), np.int8), (u, v)), shape=(n, n))
    seen = np.zeros(n, bool)
    seen[breadth_first_order(g, start, directed=True, return_predecessors=False)] = True
    return seen


def solve(hcap, vcap, src, snk):
    """-> (T bool [h,w]: reaches the sink in the residual graph of a maximum flow, S_min bool [h,w]: reached from the
    source in it, the cut value int): scipy's maximum_flow plus residual reachability."""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import maximum_flow
    h, w = hcap.shape
    n = h * w + 2
    u, v, c = _edges(hcap, vcap, src, snk)
    cap = csr_matrix((c.astype(np.int32), (u, v)), shape=(n, n))
    cap.sum_duplicates()
    res = maximum_flow(cap, n - 2, n - 1)
    r = (cap.astype(np.int64) - res.flow.tocsr().astype(np.int64)).tocoo()    # residual c(u, v) - f(u, v), f antisymmetric
    uu, vv = r.row[r.data > 0], r.col[r.data > 0]
    T = _reach(n, vv, uu, n - 1)[:h * w].reshape(h, w)                 # reverse edges: who reaches the sink
    Smin = _reach(n, uu, vv, n - 2)[:h * w].reshape(h, w)
    return T, Smin, int(res.flow_value)


def bounds(hcap, vcap, src, snk):
    """-> (smallest, largest) minimum-cut source sets, bool [h,w]."""
    T, Smin, _ = solve(hcap, vcap, src, snk)
    return Smin, ~T


def capacity(S, hcap, vcap, src, snk):
    """The capacity of the cut with source side S (bool [h,w]; the source is in S, the sink is not)."""
    S = np.asarray(S, bool)
    c = int(snk[S].sum()) + int(src[~S].sum())
    c += int(hcap[:, :-1][S[:, :-1] != S[:, 1:]].sum()) + int(vcap[:-1][S[:-1] != S[1:]].sum())
    return c


def check_certificate(hcap, vcap, src, snk, residual, T, cut):
    """Asserts that residual (int [5,h,w]: to the right, lower, left, upper neighbour and to the sink) is a preflow's
    residual graph (every edge's two residuals sum to twice its capacity and neither is negative, the sink residual lies
    in [0, snk], no pixel's excess is negative), that its flow into the sink equals the capacity of the cut (S = not T)
    and cut, and that T is exactly the set of pixels that reach the sink in it."""
    r = np.asarray(residual, np.int64)
    hcap, vcap, src, snk = (np.asarray(a, np.int64) for a in (hcap, vcap, src, snk))
    h, w = hcap.shape
    assert r.shape == (5, h, w) and (r >= 0).all()
    assert np.array_equal(r[0][:, :-1] + r[2][:, 1:], 2 * hcap[:, :-1]) and np.array_equal(r[1][:-1] + r[3][1:], 2 * vcap[:-1])
    assert not r[0][:, -1].any() and not r[2][:, 0].any() and not r[1][-1].any() and not r[3][0].any()
    assert (r[4] <= snk).all()
    out = np.zeros((h, w), np.int64)                                    # net flow out along the grid edges
    fh = hcap[:, :-1] - r[0][:, :-1]                                    # flow (x, y) -> (x + 1, y)
    fv = vcap[:-1] - r[1][:-1]
    out[:, :-1] += fh
    out[:, 1:] -= fh
    out[:-1] += fv
    out[1:] -= fv
    inflow = snk - r[4]
    assert (src - inflow - out >= 0).all()                              # no negative excess
    S = ~np.asarray(T, bool)
    assert int(inflow.sum()) == capacity(S, hcap, vcap, src, snk) == int(cut)
    idx = np.arange(h * w).reshape(h, w)
    u = [idx[:, :-1][r[0][:, :-1] > 0], idx[1:][r[3][1:] > 0], idx[:, 1:][r[2][:, 1:] > 0], idx[:-1][r[1][:-1] > 0], idx[r[4] > 0]]
    v = [idx[:, 1:][r[0][:, :-1] > 0], idx[:-1][r[3][1:] > 0], idx[:, :-1][r[2][:, 1:] > 0], idx[1:][r[1][:-1] > 0],
         np.full(int((r[4] > 0).sum()), h * w)]
    reach = _reach(h * w + 1, np.concatenate(v), np.concatenate(u), h * w)[:h * w].reshape(h, w)
    assert np.array_equal(reach, np.asarray(T, bool))


def restate(imgs, masks, tls):
    """Fed warps, masks and top-lefts -> (seam masks uint8 [h,w] each, cut values [pairs] int): the rule above."""
    out = [np.array(m, np.uint8, copy=True) for m in masks]
    cuts = []
    for i, j, rect in SM.pairs(tls, [m.shape for m in out]):
        x0, y0, x1, y1 = rect
        T, _, cut = solve(*pair_graph(imgs, out, tls, i, j, rect))
        cuts.append(cut)
        inT = T[GAP:GAP + y1 - y0, GAP:GAP + x1 - x0]
        vi = out[i][y0 - tls[i][1]:y1 - tls[i][1], x0 - tls[i][0]:x1 - tls[i][0]]
        vj = out[j][y0 - tls[j][1]:y1 - tls[j][1], x0 - tls[j][0]:x1 - tls[j][0]]
        hi, hj = vi != 0, vj != 0
        vj[~inT & hi] = 0
        vi[inT & hj] = 0
    return out, cuts


def _with_gc_seams(reference, frames, M, Hc, Wc, *args):
    """oracle/seam's end-to-end reference (multiband or feather) fed restate's seams in place of cv2's Voronoi seams.
    oracle/seam's references take the seams from its finder, cv2_seams(masks, tls); that finder is stood in for, for the
    length of the call, by restate's seams of the same fed masks, computed from the uncompensated 3-channel warps (a
    1-channel frame repeated), the graph-cut finder's input."""
    rgb = [f if f.ndim == 3 and f.shape[2] == 3 else np.repeat(f.reshape(f.shape[0], f.shape[1], 1), 3, 2) for f in frames]
    _, imgs, masks, tls = EX.fed(rgb, M, Hc, Wc)
    seams, _ = restate(imgs, masks, tls)

    def finder(m, t):
        assert _equal(m, masks) and list(t) == list(tls), "oracle/seam fed other masks than the graph-cut seams were cut on"
        return [s.copy() for s in seams]
    voronoi = SM.cv2_seams
    SM.cv2_seams = finder
    try:
        return reference(frames, M, Hc, Wc, *args)
    finally:
        SM.cv2_seams = voronoi


def _equal(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


def multiband(frames, M, Hc, Wc, bands, gains=None):
    """oracle/seam.multiband with restate's seams: -> (mosaic uint8 [Hc,Wc,3], mask uint8 [Hc,Wc])."""
    return _with_gc_seams(SM.multiband, frames, M, Hc, Wc, bands, gains)


def feather(frames, M, Hc, Wc, feather_px, gains=None):
    """oracle/seam.feather with restate's seams (cut on the 3-channel frames, a 1-channel frame repeated)."""
    return _with_gc_seams(SM.feather, frames, M, Hc, Wc, feather_px, gains)
