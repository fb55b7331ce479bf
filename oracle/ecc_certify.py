"""Float64 certification of one ECC iteration (csrc/ecc.cu) on the kernels' own gates.  Test-only: no GPU.

The per-pixel gates are restated bit for bit:
  - the warp map (ecc_map): the products M[k] * x of a float32 entry and an integer below 2^15 are exact in fp64, so
    X0, Y0, W0 round only in their two additions, in source order, whichever contraction ptxas picks; 32 / W0, the
    products with it and the rounding half to even are single IEEE operations.  No coordinate is left ambiguous;
  - the INTER_NEAREST mask, the footprint test, and iw, gx, gy through ecc_bilerp's explicitly rounded operations;
  - iz = iw - float(mean I), tz = T - float(mean T), with the means from the kernel's fp64 totals.
The 53 Jacobian / Hessian terms of ecc_jacobian_px are then evaluated in fp64 with a bound on the distance of the
kernel's fp32 value from them: every operation of the fp32 sequence (den, hatX / hatY, gxd / gyd, tmp, J, the product
that is added) is charged u = 2^-24 of its magnitude plus the propagated bounds of its operands.  Charging a rounding to
every operation covers every FMA contraction, since a fused operation rounds once where the bound charges twice.  The fp64
evaluation is charged the same with 2^-53, so the bound is on |kernel - oracle|.

`solve` restates ecc_solve_update / lu_solve2_warp in fp64 with fma emulated exactly (fractions.Fraction), from the 53
sums and the 5 moments, and applies the float32 update.
"""
import math
from fractions import Fraction

import numpy as np

from . import ecc as E

U32 = 2.0 ** -24
U64 = 2.0 ** -53
TINY32 = 2.0 ** -149                     # an underflowing fp32 operation is off by at most this much
NACC = 53
SPLIT_TILE = 16384                       # kEccSplitTile: 256 threads x 64 pixels
SPLIT_THREADS = 256
SPLIT_PX_PER_THREAD = 64
ONE_CTA_THREADS_Y, ONE_CTA_THREADS_X = 16, 32   # ecc_iterate_kernel: warp w takes rows w, w + 16, ...; lane l columns l, l + 32, ...
SLOT = (0, 3, 6, 1, 4, 7, 2, 5)          # update_warping_matrix_ECC's parameter order
TREE_ULPS = 16                           # fp64 additions a value passes through in a CTA's butterfly + warp sum, rounded up
_INT_MIN, _INT_MAX = float(np.iinfo(np.int32).min), float(np.iinfo(np.int32).max)


def upper_index():
    """(r, c) of each of the 36 Hessian sums, row by row over the upper triangle."""
    return [(r, c) for r in range(8) for c in range(r, 8)]


def one_cta_px_per_thread(H, Wd):
    return -(-H // ONE_CTA_THREADS_Y) * -(-Wd // ONE_CTA_THREADS_X)


# ---------------------------------------------------------------------------- gates
def gates(Wf, Tb, Ib, o0=0, o1=None):
    """The kernel's per-pixel gates for the row-major pixels [o0, o1) of the plane under the float32 W.
    -> dict x, y (int64), inside (footprint touches the image), mask, iw, gx, gy, t (float32)."""
    H, Wd = Tb.shape
    o1 = H * Wd if o1 is None else o1
    o = np.arange(o0, o1, dtype=np.int64)
    y = o // Wd; x = o - y * Wd
    M = np.asarray(Wf, np.float32).astype(np.float64).reshape(9)
    xd, yd = x.astype(np.float64), y.astype(np.float64)
    X0 = (M[0] * xd + M[1] * yd) + M[2]
    Y0 = (M[3] * xd + M[4] * yd) + M[5]
    W0 = (M[6] * xd + M[7] * yd) + M[8]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        wl = np.where(W0 != 0, 32.0 / W0, 0.0)
        wn = np.where(W0 != 0, 1.0 / W0, 0.0)
        q = lambda v: np.rint(np.clip(v, _INT_MIN, _INT_MAX)).astype(np.int64)
        X, Y, Xn, Yn = q(X0 * wl), q(Y0 * wl), q(X0 * wn), q(Y0 * wn)
    xi = np.clip(X >> 5, -32768, 32767); yi = np.clip(Y >> 5, -32768, 32767)
    ax = (X & 31).astype(np.float32) * np.float32(1.0 / 32.0); ay = (Y & 31).astype(np.float32) * np.float32(1.0 / 32.0)
    mask = (Xn >= 0) & (Xn < Wd) & (Yn >= 0) & (Yn < H)
    inside = ~((xi + 1 < 0) | (xi >= Wd) | (yi + 1 < 0) | (yi >= H))
    gxp, gyp = E.gradients(Ib)
    return dict(x=x, y=y, inside=inside, mask=mask, iw=E.bilinear(Ib, xi, yi, ax, ay), gx=E.bilinear(gxp, xi, yi, ax, ay),
                gy=E.bilinear(gyp, xi, yi, ax, ay), t=Tb.reshape(-1)[o0:o1].astype(np.float32))


def moments_px(g):
    """Per pixel the 5 pass-1 terms (n, Iw, Iw^2, T, T^2) as fp64 (all exact: the squares of fp32 values fit in fp64)."""
    m = g["mask"]
    iw, t = g["iw"].astype(np.float64), g["t"].astype(np.float64)
    z = np.zeros_like(iw)
    return np.stack([m.astype(np.float64), np.where(m, iw, z), np.where(m, iw * iw, z), np.where(m, t, z), np.where(m, t * t, z)], 1)


def means_f32(tot):
    """ecc_moments' float32 means from the 5 fp64 totals."""
    n = tot[0]
    mI = tot[1] / n if n > 0 else 0.0
    mT = tot[3] / n if n > 0 else 0.0
    return np.float32(mI), np.float32(mT)


def add_tiles(slab):
    """The kernels' fp64 total of per-tile sums [nt, k], added in tile order."""
    tot = np.zeros(slab.shape[1])
    for t in range(slab.shape[0]):
        tot = tot + slab[t]
    return tot


# ---------------------------------------------------------------------------- the 53 terms and their bounds
def _mul(a, b, u, tiny):
    (va, ea), (vb, eb) = a, b
    v = va * vb
    e = np.abs(va) * eb + np.abs(vb) * ea + ea * eb
    return v, e + u * (np.abs(v) + e) + tiny


def _add(a, b, u, tiny):
    (va, ea), (vb, eb) = a, b
    v = va + vb
    e = ea + eb
    return v, e + u * (np.abs(v) + e) + tiny


def _neg(a):
    return -a[0], a[1]


def _div(a, b, u, tiny):
    (va, ea), (vb, eb) = a, b
    ab = np.abs(vb)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        v = va / vb
        e = np.where(ab > eb, (ea * ab + np.abs(va) * eb) / (ab * (ab - eb)), np.inf)
    return v, e + u * (np.abs(v) + e) + tiny


def _sequence(x, y, h, gx, gy, iz, tz, u, tiny):
    """ecc_jacobian_px's operations in its order, each value with its bound: -> (terms [N,53], bounds [N,53])."""
    z = np.zeros_like(gx)
    ex = lambda v: (np.asarray(v, np.float64) + z, z)                  # exact inputs
    xf, yf = ex(x), ex(y)
    hh = [ex(np.float64(v)) for v in h]
    m = lambda a, b: _mul(a, b, u, tiny)
    a = lambda p, q: _add(p, q, u, tiny)
    d = lambda p, q: _div(p, q, u, tiny)
    den = a(a(m(xf, hh[2]), m(yf, hh[5])), ex(1.0))
    numX = a(a(_neg(m(xf, hh[0])), _neg(m(yf, hh[3]))), _neg(hh[6]))
    numY = a(a(_neg(m(xf, hh[1])), _neg(m(yf, hh[4]))), _neg(hh[7]))
    hatX, hatY = d(numX, den), d(numY, den)
    gxd, gyd = d(ex(gx), den), d(ex(gy), den)
    tmp = a(m(hatX, gxd), m(hatY, gyd))
    J = [m(gxd, xf), m(gyd, xf), m(tmp, xf), m(gxd, yf), m(gyd, yf), m(tmp, yf), gxd, gyd]
    izv, tzv = ex(iz), ex(tz)
    terms = [m(J[r], J[c]) for r, c in upper_index()] + [m(J[r], izv) for r in range(8)] + [m(J[r], tzv) for r in range(8)]
    terms.append(m(tzv, izv))
    return np.stack([t[0] for t in terms], 1), np.stack([t[1] for t in terms], 1)


def h8(Wf):
    """The parameter-order entries ecc_jacobian_px reads: W[0], W[3], W[6], W[1], W[4], W[7], W[2], W[5] (float32)."""
    w = np.asarray(Wf, np.float32).reshape(9)
    return [w[k] for k in (0, 3, 6, 1, 4, 7, 2, 5)]


def jacobian_terms(g, Wf, mIf, mTf):
    """Pixels whose footprint touches the image: -> (sel index array, terms [n,53] fp64, bounds [n,53] on
    |kernel fp32 term - terms|)."""
    sel = np.nonzero(g["inside"])[0]
    m = g["mask"][sel]
    iw = g["iw"][sel]
    iz = np.where(m, iw - np.float32(mIf), iw).astype(np.float32)
    tz = np.where(m, g["t"][sel] - np.float32(mTf), np.float32(0)).astype(np.float32)
    args = (g["x"][sel], g["y"][sel], h8(Wf), g["gx"][sel].astype(np.float64), g["gy"][sel].astype(np.float64),
            iz.astype(np.float64), tz.astype(np.float64))
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        t64, e32 = _sequence(*args, u=U32, tiny=TINY32)
        _, e64 = _sequence(*args, u=U64, tiny=0.0)
    return sel, t64, (e32 + e64) * (1.0 + 1e-6)


def sum_bound(terms, bounds, k):
    """Bound on |a kernel sum of these terms - their exact fp64 sum| when each thread adds at most k of them in fp32 and the
    threads' partials meet in an fp64 tree; also charges the oracle's own fp64 summation."""
    a = np.abs(terms).sum(0)
    return bounds.sum(0) + (k - 1) * U32 * 1.01 * (a + bounds.sum(0)) + (TREE_ULPS + math.log2(max(len(terms), 2)) + 2) * U64 * a


# ---------------------------------------------------------------------------- the solve
def fma(a, b, c):
    """a * b + c rounded once (Python 3.12 has no math.fma)."""
    if not (math.isfinite(a) and math.isfinite(b) and math.isfinite(c)):
        return a * b + c
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def lu_solve2(A, b0, b1):
    """lu_solve2_warp: partial pivoting (the first row of maximal |a_k|), fma elimination, back substitution."""
    a = [[float(A[r][c]) for c in range(8)] + [float(b0[r]), float(b1[r])] for r in range(8)]
    for k in range(8):
        piv = k
        for r in range(k + 1, 8):
            if abs(a[r][k]) > abs(a[piv][k]):
                piv = r
        a[k], a[piv] = a[piv], a[k]
        pk = a[k]
        for r in range(k + 1, 8):
            f = a[r][k] / pk[k] if pk[k] != 0 else math.copysign(math.inf, a[r][k]) if a[r][k] != 0 else math.nan
            for c in range(k + 1, 10):
                a[r][c] = fma(-f, pk[c], a[r][c])
            a[r][k] = 0.0
    x0, x1 = [0.0] * 8, [0.0] * 8
    for k in range(7, -1, -1):
        dk = a[k][k]
        x0[k] = a[k][8] / dk if dk != 0 else math.nan
        x1[k] = a[k][9] / dk if dk != 0 else math.nan
        for r in range(k):
            a[r][8] = fma(-a[r][k], x0[k], a[r][8])
            a[r][9] = fma(-a[r][k], x1[k], a[r][9])
    return x0, x1


def _norms(mom, fused):
    n = mom[0]
    if not n > 0:
        return 0.0, 0.0
    out = []
    for s1, s2 in ((mom[1], mom[2]), (mom[3], mom[4])):
        m = s1 / n
        v = fma(-m, m, s2 / n) if fused else s2 / n - m * m
        sd = math.sqrt(max(v, 0.0))
        out.append(math.sqrt(n * sd * sd))
    return out[0], out[1]


def solve(tot, mom, Wf, fused=True):
    """ecc_solve_update from the 53 sums and the 5 moments: -> dict(W float32 [9], rho, lambda_d, status, and the
    condition number cond of the Hessian scaled to a unit diagonal).  `fused`
    picks fma for every contraction the compiler may make (the moments' variance, ipH / tpH, lambda_n, dp) or none."""
    tot = [float(v) for v in tot]
    imgNorm, tmpNorm = _norms([float(v) for v in mom], fused)
    corr = tot[52]
    with np.errstate(divide="ignore", invalid="ignore"):
        rho = float(np.float64(corr) / np.float64(imgNorm * tmpNorm))
    A = [[0.0] * 8 for _ in range(8)]
    for q, (r, c) in enumerate(upper_index()):
        A[r][c] = A[c][r] = tot[q]
    xi, xt = lu_solve2(A, tot[36:44], tot[44:52])
    ipH = tpH = 0.0
    for k in range(8):
        if fused:
            ipH, tpH = fma(tot[36 + k], xi[k], ipH), fma(tot[44 + k], xi[k], tpH)
        else:
            ipH, tpH = ipH + tot[36 + k] * xi[k], tpH + tot[44 + k] * xi[k]
    lambda_n = fma(imgNorm, imgNorm, -ipH) if fused else imgNorm * imgNorm - ipH
    lambda_d = corr - tpH
    status = E.ECC_OK
    if math.isnan(rho):
        status = E.ECC_NAN
    elif lambda_d <= 0.0:
        status = E.ECC_NOCONV
    W = np.asarray(Wf, np.float32).reshape(9).copy()
    if status == E.ECC_OK:
        lam = lambda_n / lambda_d if lambda_d != 0 else math.nan
        for k in range(8):
            dp = np.float32(fma(lam, xt[k], -xi[k]) if fused else lam * xt[k] - xi[k])
            W[SLOT[k]] = np.float32(W[SLOT[k]] + dp)
    with np.errstate(all="ignore"):
        A = np.array(A)
        d = np.sqrt(np.abs(np.diag(A)))
        ok = np.all(np.isfinite(A)) and np.all(d > 0)
        cond = float(np.linalg.cond(A / d[:, None] / d[None, :])) if ok else math.inf
    return dict(W=W, rho=rho, lambda_d=lambda_d, lambda_n=lambda_n, corr=corr, tpH=tpH, status=status, cond=cond)


def solve_fp64(tot, mom, Wf):
    """The same solve without the update's float32 rounding: the fp64 W + dp (for sensitivities)."""
    tot = [float(v) for v in tot]
    imgNorm, tmpNorm = _norms([float(v) for v in mom], False)
    A = np.zeros((8, 8))
    for q, (r, c) in enumerate(upper_index()):
        A[r, c] = A[c, r] = tot[q]
    try:
        sol = np.linalg.solve(A, np.stack([tot[36:44], tot[44:52]], 1))
    except np.linalg.LinAlgError:
        return np.full(9, np.nan)
    lam = (imgNorm * imgNorm - float(np.dot(tot[36:44], sol[:, 0]))) / (tot[52] - float(np.dot(tot[44:52], sol[:, 0])))
    W = np.asarray(Wf, np.float32).astype(np.float64).reshape(9).copy()
    for k in range(8):
        W[SLOT[k]] += lam * sol[k, 1] - sol[k, 0]
    return W


def w_bound(tot, mom, Wf, b_tot, b_mom):
    """First-order bound on |W(kernel sums) - W(exact sums)| per entry: the solve's sensitivity to each of the 53 + 5
    sums (central differences in fp64) times that sum's bound, doubled, plus the float32 rounding of the update."""
    tot = np.asarray(tot, np.float64); mom = np.asarray(mom, np.float64)
    out = np.zeros(9)
    for vec, bnd, which in ((tot, b_tot, 0), (mom, b_mom, 1)):
        for k in range(len(vec)):
            if k == 0 and which == 1:
                continue                                                   # n is an exact count
            h = max(abs(vec[k]) * 1e-7, bnd[k], 1e-300)
            p, m_ = vec.copy(), vec.copy()
            p[k] += h; m_[k] -= h
            args_p = (p, mom) if which == 0 else (tot, p)
            args_m = (m_, mom) if which == 0 else (tot, m_)
            s = (solve_fp64(*args_p, Wf) - solve_fp64(*args_m, Wf)) / (2 * h)
            out += np.abs(s) * bnd[k]
    W = solve_fp64(tot, mom, Wf)
    return 2.0 * out + 2.0 * np.abs(W) * U32 + 2.0 * np.abs(W - np.asarray(Wf, np.float32).astype(np.float64).reshape(9)) * U32
