"""CPU tests of the ECC certification's ground: the blur's BORDER_REFLECT_101 index (compiled from csrc/common.cuh) against
cv2.borderInterpolate, oracle/ecc_certify.py's per-pixel bound against exact evaluation of every FMA contraction of
ecc_jacobian_px, its terms against oracle/ecc.py's sums, and its exact-fma solve against np.linalg.solve."""
import itertools
import math
import os
import shutil
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
cv2 = pytest.importorskip("cv2")
import _ecc_kinds as K  # noqa: E402
from oracle import ecc as E  # noqa: E402
from oracle import ecc_certify as C  # noqa: E402

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NEEDS_NVCC = pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="the CUDA toolkit is not installed")

_DRIVER = r"""
#include <cstdio>
#include "common.cuh"
int main() {
  for (int n = 2; n <= 9; ++n) {
    for (int i = -2; i <= n + 1; ++i) printf("%d ", udh::reflect101(i, n));
    printf("\n");
  }
  return 0;
}
"""


@NEEDS_NVCC
def test_reflect101_is_cv2_border_reflect_101(tmp_path):
    from unsuperviseddeephomographyral2018_b200 import build_ext
    src = tmp_path / "reflect.cu"
    src.write_text(_DRIVER)
    exe = str(tmp_path / "reflect")
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    p = subprocess.run([nvcc, "-std=c++17", "-I", build_ext.CSRC, str(src), "-o", exe], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600)
    assert p.returncode == 0, p.stdout
    rows = subprocess.run([exe], stdout=subprocess.PIPE, text=True, check=True, timeout=60).stdout.splitlines()
    for n, row in zip(range(2, 10), rows):
        want = [cv2.borderInterpolate(i, n, cv2.BORDER_REFLECT_101) for i in range(-2, n + 2)]
        assert [int(v) for v in row.split()] == want, n
    # the single reflection it replaces read outside a plane of side 2
    old = lambda i, n: -i if i < 0 else (2 * n - 2 - i if i >= n else i)
    assert [old(i, 2) for i in range(-2, 4)] == [2, 1, 0, 1, 0, -1]
    assert [cv2.borderInterpolate(i, 2, cv2.BORDER_REFLECT_101) for i in range(-2, 4)] == [0, 1, 0, 1, 0, 1]


def test_oracle_blur_is_cv2_gaussian_at_small_sides():
    rng = np.random.default_rng(3)
    for h, w in ((2, 2), (2, 7), (7, 2), (3, 3), (3, 5), (4, 4), (5, 9)):
        u8 = rng.integers(0, 256, (h, w), dtype=np.uint8)
        assert np.array_equal(E.blur(u8), cv2.GaussianBlur(u8.astype(np.float32), (5, 5), 0, 0)), (h, w)


# ---- the per-pixel bound against exact evaluation -------------------------------------------------------------------------
def rn32(q):
    """The float32 nearest to the rational q, ties to even, as a Fraction."""
    if q == 0:
        return Fraction(0)
    f = np.float32(float(q))
    best = None
    for c in (np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))):
        d = abs(Fraction(float(c)) - q)
        if best is None or d < best[0] or (d == best[0] and int(np.array(c, np.float32).view(np.uint32)) % 2 == 0):
            best = (d, c)
    return Fraction(float(best[1]))


def _pair_sum(a, b, c, d, how):
    """a b + c d in fp32: no contraction (0), fma(a, b, rn(c d)) (1) or fma(c, d, rn(a b)) (2)."""
    if how == 0:
        return rn32(rn32(a * b) + rn32(c * d))
    if how == 1:
        return rn32(a * b + rn32(c * d))
    return rn32(rn32(a * b) + c * d)


def kernel_terms_exact(x, y, h, gx, gy, iz, tz, how):
    """ecc_jacobian_px's fp32 sequence with the contraction choices how = (den, hatX, hatY, tmp): -> the 53 terms, each
    rounded to fp32 (a separate multiply) and exact (fused into the accumulating fma)."""
    F = lambda v: Fraction(float(v))
    x, y, gx, gy, iz, tz = F(x), F(y), F(gx), F(gy), F(iz), F(tz)
    h = [F(v) for v in h]
    den = rn32(_pair_sum(x, h[2], y, h[5], how[0]) + 1)
    hatX = rn32(rn32(_pair_sum(-x, h[0], -y, h[3], how[1]) - h[6]) / den)
    hatY = rn32(rn32(_pair_sum(-x, h[1], -y, h[4], how[2]) - h[7]) / den)
    gxd, gyd = rn32(gx / den), rn32(gy / den)
    tmp = _pair_sum(hatX, gxd, hatY, gyd, how[3])
    J = [rn32(gxd * x), rn32(gyd * x), rn32(tmp * x), rn32(gxd * y), rn32(gyd * y), rn32(tmp * y), gxd, gyd]
    prods = [J[r] * J[c] for r, c in C.upper_index()] + [J[r] * iz for r in range(8)] + [J[r] * tz for r in range(8)] + [tz * iz]
    return prods, [rn32(p) for p in prods]


@pytest.mark.parametrize("kind", ["identity", "fraction", "perturbed", "horizon", "handful", "saturate"])
def test_per_pixel_bound_holds_for_every_contraction(kind):
    h, w = 48, 200
    T, Im, Wf = K.case(kind, h, w, seed=5)
    Tb, Ib = E.blur(T), E.blur(Im)
    g = C.gates(Wf, Tb, Ib)
    mom = C.moments_px(g).sum(0)
    mIf, mTf = C.means_f32(mom)
    sel, t64, bnd = C.jacobian_terms(g, Wf, mIf, mTf)
    ok = np.all(np.isfinite(t64), 1) & np.all(np.isfinite(bnd), 1)
    idx = np.nonzero(ok)[0]
    assert len(idx) > 0
    pick = np.unique(np.r_[idx[:2], idx[-2:], np.random.default_rng(1).choice(idx, min(6, len(idx)), replace=False)])
    if kind == "horizon":                               # the wl = 0 pixel and its neighbours
        pick = np.unique(np.r_[pick, [i for i in idx if g["x"][sel[i]] in (127, 128, 129, 161)][:6]])
    worst = 0.0
    for i in pick:
        p = sel[i]
        m = bool(g["mask"][p])
        iz = np.float32(g["iw"][p] - mIf) if m else g["iw"][p]
        tz = np.float32(g["t"][p] - mTf) if m else np.float32(0)
        for how in itertools.product(range(3), repeat=4):
            for vals in kernel_terms_exact(g["x"][p], g["y"][p], C.h8(Wf), g["gx"][p], g["gy"][p], iz, tz, how):
                err = np.array([abs(float(v - Fraction(float(t)))) for v, t in zip(vals, t64[i])])
                assert np.all(err <= bnd[i]), (kind, p, how, np.nonzero(err > bnd[i]))
                r = err / np.where(bnd[i] > 0, bnd[i], 1.0)
                worst = max(worst, float(r.max()))
    print("%s: %d pixels x 81 contractions, worst error / bound %.3f" % (kind, len(pick), worst))


@pytest.mark.parametrize("kind", ["identity", "fraction", "perturbed", "horizon"])
def test_oracle_terms_sum_to_the_restatement_sums(kind):
    """The per-pixel terms over a plane give oracle/ecc.py's Hessian, projections and correlation after one iteration, to
    within the terms' bounds (oracle/ecc.py evaluates the same fp32 sequence without contraction)."""
    h, w = 96, 200
    T, Im, Wf = K.case(kind, h, w, seed=7)
    trace = []
    E.ecc(T, Im, Wf, max_iters=1, trace=trace)
    g = C.gates(Wf, E.blur(T), E.blur(Im))
    mom = C.moments_px(g).sum(0)
    mIf, mTf = C.means_f32(mom)
    sel, t64, bnd = C.jacobian_terms(g, Wf, mIf, mTf)
    tot = t64.sum(0)
    tr = trace[0]
    ref = np.r_[[tr["hessian"][r, c] for r, c in C.upper_index()], tr["ip"], tr["tp"], tr["corr"]]
    slack = bnd.sum(0) + 64 * C.U64 * np.abs(t64).sum(0)
    assert np.all(np.abs(tot - ref) <= slack), np.abs(tot - ref) / slack
    print("%s: worst |sum - oracle/ecc.py| / bound %.3e" % (kind, float((np.abs(tot - ref) / slack).max())))


def test_fma_is_exact():
    a, b, c = 1.0 + 2.0 ** -30, 1.0 - 2.0 ** -30, -1.0
    assert C.fma(a, b, c) == -(2.0 ** -60) and a * b + c == 0.0


def test_lu_solve2_agrees_with_numpy_to_the_condition_number():
    rng = np.random.default_rng(11)
    systems = []
    for s in range(6):
        J = rng.standard_normal((8, 200)) * np.logspace(0, s, 8)[:, None]
        systems.append((J @ J.T, rng.standard_normal(8), rng.standard_normal(8)))
    T, Im, Wf = K.case("perturbed", 64, 96, seed=2)
    trace = []
    E.ecc(T, Im, Wf, max_iters=1, trace=trace)
    systems.append((trace[0]["hessian"], trace[0]["ip"], trace[0]["tp"]))
    for A, b0, b1 in systems:
        x0, x1 = C.lu_solve2(A.tolist(), b0, b1)
        ref = np.linalg.solve(A, np.stack([b0, b1], 1))
        cond = np.linalg.cond(A)
        for got, want in ((x0, ref[:, 0]), (x1, ref[:, 1])):
            rel = np.abs(np.array(got) - want).max() / np.abs(want).max()
            assert rel <= 16 * cond * 2.0 ** -52, (rel, cond)
