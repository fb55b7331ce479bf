"""GPU certification of both ECC kernels (csrc/ecc.cu) against float64 on their own gates (oracle/ecc_certify.py):
the blurred planes against cv2.GaussianBlur, the split kernel's per-tile moments and 53 Jacobian / Hessian sums, its solve
from its own totals, both kernels' W after one iteration against the float64 truth within a bound propagated from the
sums, and the iteration state and stopping rule.  The workspace layout comes from udh_debug_ecc_layout."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
cv2 = pytest.importorskip("cv2")
import _ecc_kinds as K  # noqa: E402
from oracle import ecc as E  # noqa: E402
from oracle import ecc_certify as C  # noqa: E402

pytestmark = pytest.mark.gpu
KERNELS = ("one_cta", "split")
WORST = {}


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _note(section, r):
    WORST[section] = max(WORST.get(section, 0.0), float(r))
    print("worst ratio so far, %s: %.3e" % (section, WORST[section]))


def layout(B, H, Wd):
    from unsuperviseddeephomographyral2018_b200._lib import check, lib
    off, nt = (ctypes.c_size_t * 4)(), ctypes.c_int()
    check(lib.udh_debug_ecc_layout(B, H, Wd, off, ctypes.byref(nt)), "udh_debug_ecc_layout")
    return list(off), nt.value


def run(kernel, T, Im, W0, iters, eps=0.0):
    """-> dict(W [B,9], rho, iters, status, blurred [2,B,H,W], and for the split kernel slab1 [B,nt,5], slab2 [B,nt,53])."""
    from unsuperviseddeephomographyral2018_b200._lib import check, lib
    T, Im = np.ascontiguousarray(T), np.ascontiguousarray(Im)
    B, H, Wd = T.shape
    fn, wsf = (("udh_ecc_homography_split", "udh_ecc_split_workspace_bytes") if kernel == "split"
               else ("udh_ecc_homography", "udh_ecc_workspace_bytes"))
    nbytes = getattr(lib, wsf)(B, H, Wd)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    dT, dI = torch.from_numpy(T).cuda(), torch.from_numpy(Im).cuda()
    dW0 = torch.from_numpy(np.ascontiguousarray(np.asarray(W0, np.float32).reshape(B, 9))).cuda()
    W = torch.empty(B, 9, dtype=torch.float32, device="cuda")
    rho = torch.empty(B, dtype=torch.float64, device="cuda")
    it = torch.empty(B, dtype=torch.int32, device="cuda")
    st = torch.empty(B, dtype=torch.int32, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    check(getattr(lib, fn)(p(dT), p(dI), p(dW0), int(iters), float(eps), p(W), p(rho), p(it), p(st), p(ws), nbytes, B, H, Wd,
                           ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), fn)
    torch.cuda.synchronize()
    off, nt = layout(B, H, Wd)
    raw = ws.cpu().numpy()
    npx = B * H * Wd
    out = dict(W=W.cpu().numpy(), rho=rho.cpu().numpy(), iters=it.cpu().numpy(), status=st.cpu().numpy(),
               blurred=raw[off[0]:off[0] + 8 * npx].view(np.float32).reshape(2, B, H, Wd))
    if kernel == "split":
        out["slab1"] = raw[off[2]:off[2] + B * nt * 5 * 8].view(np.float64).reshape(B, nt, 5)
        out["slab2"] = raw[off[3]:off[3] + B * nt * C.NACC * 8].view(np.float64).reshape(B, nt, C.NACC)
    return out


# ---- A. blur ------------------------------------------------------------------------------------------------------------
BLUR_SHAPES = [(2, 2), (2, 7), (7, 2), (3, 3), (3, 5), (4, 4), (5, 9), (16, 22), (113, 145), (128, 128), (240, 320), (375, 500),
               (1080, 1920), (3000, 4000), (2, 32767), (32767, 2)]


@pytest.mark.parametrize("h,w", BLUR_SHAPES)
def test_blur_is_bit_identical_to_cv2(h, w):
    """Both kernels' blurred planes equal cv2.GaussianBlur(float32(u8), (5, 5), 0, 0) (BORDER_REFLECT_101), alone and in a
    batch of three different pairs, so a read across a plane's border into its neighbour would show."""
    _need_gpu()
    rng = np.random.default_rng(h * 40000 + w)
    T = rng.integers(0, 256, (3, h, w), dtype=np.uint8)
    Im = rng.integers(0, 256, (3, h, w), dtype=np.uint8)
    W0 = np.tile(np.eye(3, dtype=np.float32), (3, 1, 1))
    ref = [[cv2.GaussianBlur(P[b].astype(np.float32), (5, 5), 0, 0) for b in range(3)] for P in (T, Im)]
    for kernel in KERNELS:
        for B in (1, 3):
            got = run(kernel, T[:B], Im[:B], W0[:B], 0)["blurred"]
            for z in range(2):
                for b in range(B):
                    assert np.array_equal(got[z, b], ref[z][b]), (kernel, B, z, b)


# ---- B, C, D. the split kernel's sums and solve ----------------------------------------------------------------------------
SPLIT_CASES = ([((240, 320), k) for k in K.KINDS] +
               [((h, w), k) for (h, w) in ((2, 2), (2, 7), (3, 5), (16, 22), (113, 145), (128, 128), (375, 500))
                for k in ("identity", "fraction", "handful")] +
               [((128, 128), "perturbed"), ((375, 500), "perturbed"), ((375, 500), "horizon"), ((375, 500), "saturate"),
                ((1080, 1920), "perturbed"), ((1080, 1920), "horizon")])


def _tiles_to_check(nt, mask_tiles):
    if nt <= 8:
        return list(range(nt))
    return sorted(set([0, 1, nt // 3, nt // 2, nt - 2, nt - 1] + mask_tiles[:4]))


@pytest.mark.parametrize("shape,kind", SPLIT_CASES, ids=["%dx%d-%s" % (s[0], s[1], k) for s, k in SPLIT_CASES])
def test_split_sums_and_solve_against_float64(shape, kind):
    """B: per tile, n equals the restated mask count and the four moment sums agree to 100 * 2^-53 of their magnitude.
    C: every checked tile's 53 sums are within the bound derived from the fp32 sequence (64 px per thread).
    D: W after one iteration is the exact restatement of the solve from the kernel's own totals, within 1 fp32 ulp per
    entry; rho within its fp64 bound; the status is the rule's."""
    _need_gpu()
    h, w = shape
    T, Im, Wf = K.case(kind, h, w, seed=1)
    out = run("split", T[None], Im[None], Wf[None], 1)
    Tb, Ib = out["blurred"][0, 0], out["blurred"][1, 0]
    assert np.array_equal(Tb, E.blur(T)) and np.array_equal(Ib, E.blur(Im))
    slab1, slab2 = out["slab1"][0], out["slab2"][0]
    nt = slab1.shape[0]
    mom = C.add_tiles(slab1)
    mIf, mTf = C.means_f32(mom)
    _, _, _, _, mask_all = E.warp_map(Wf, h, w)
    mflat = mask_all.reshape(-1)
    edge = [t for t in range(nt) if 0 < mflat[t * C.SPLIT_TILE:(t + 1) * C.SPLIT_TILE].sum() < len(mflat[t * C.SPLIT_TILE:(t + 1) * C.SPLIT_TILE])]
    worst_b = worst_c = 0.0
    for t in _tiles_to_check(nt, edge):
        o0, o1 = t * C.SPLIT_TILE, min(h * w, (t + 1) * C.SPLIT_TILE)
        g = C.gates(Wf, Tb, Ib, o0, o1)
        mp = C.moments_px(g)
        assert slab1[t, 0] == mp[:, 0].sum(), (t, slab1[t, 0], mp[:, 0].sum())
        for k in range(1, 5):
            ref = math.fsum(mp[:, k])
            tol = 100 * C.U64 * np.abs(mp[:, k]).sum()
            assert abs(slab1[t, k] - ref) <= tol, (t, k, slab1[t, k], ref)
            worst_b = max(worst_b, abs(slab1[t, k] - ref) / tol if tol > 0 else 0.0)
        if kind == "den0":
            continue                                                      # inf / NaN terms where den = 0: status only
        _, t64, bnd = C.jacobian_terms(g, Wf, mIf, mTf)
        ref = np.array([math.fsum(t64[:, k]) for k in range(C.NACC)])
        b = C.sum_bound(t64, bnd, C.SPLIT_PX_PER_THREAD)
        diff = np.abs(slab2[t] - ref)
        assert np.all(diff <= b), (t, np.nonzero(diff > b), diff[diff > b], b[diff > b])
        worst_c = max(worst_c, float(np.max(np.where(b > 0, diff / np.where(b > 0, b, 1), 0))))
    _note("B moments / (100 * 2^-53 sum)", worst_b)
    _note("C jacobian sums / derived bound", worst_c)
    # D: the solve from the kernel's own totals
    tot = C.add_tiles(slab2)
    fused, plain = C.solve(tot, mom, Wf, fused=True), C.solve(tot, mom, Wf, fused=False)
    Wk = out["W"][0]
    if fused["status"] == E.ECC_OK and np.all(np.isfinite(fused["W"])) and fused["cond"] < 1e10:
        ulp = lambda a, b: np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))
        ulps = np.minimum(ulp(Wk, fused["W"]), ulp(Wk, plain["W"]))
        assert ulps.max() <= 1, (Wk, fused["W"], plain["W"])
        _note("D W ulps from the exact solve", ulps.max())
        print("%s %dx%d: %d of 9 entries bit-identical to the restated solve" % (kind, h, w, int((ulps == 0).sum())))
    rho_b = abs(fused["rho"] - plain["rho"]) + 8 * C.U64 * abs(fused["rho"])
    if not math.isnan(fused["rho"]):
        assert abs(out["rho"][0] - fused["rho"]) <= rho_b, (out["rho"][0], fused["rho"])
    else:
        assert math.isnan(out["rho"][0])
    ld_b = abs(fused["lambda_d"] - plain["lambda_d"]) + 64 * C.U64 * (abs(fused["corr"]) + abs(fused["tpH"]))
    if not abs(fused["lambda_d"]) <= ld_b and fused["cond"] < 1e10:
        assert out["status"][0] == fused["status"], (out["status"][0], fused)
    assert out["iters"][0] == 1
    if kind in ("none", "flat"):
        assert out["status"][0] == E.ECC_NAN and np.array_equal(Wk, Wf.reshape(9))


# ---- E. both kernels against the float64 truth -----------------------------------------------------------------------------
def _truth(T, Im, Wf, k, nt):
    """The exact-sum solve and the bound on |W_kernel - W_truth| for a kernel whose threads add k pixels each."""
    Tb, Ib = E.blur(T), E.blur(Im)
    g = C.gates(Wf, Tb, Ib)
    mp = C.moments_px(g)
    mom = np.array([math.fsum(mp[:, j]) for j in range(5)])
    n = mom[0]
    if n > 0:                                  # float(mean) must not sit on a float32 rounding boundary
        for s in (1, 3):
            m = mom[s] / n
            if np.float32(m * (1 + 1e-12)) != np.float32(m * (1 - 1e-12)):
                return None
    mIf, mTf = C.means_f32(mom)
    _, t64, bnd = C.jacobian_terms(g, Wf, mIf, mTf)
    tot = np.array([math.fsum(t64[:, j]) for j in range(C.NACC)])
    if not np.isfinite(t64).all():
        return C.solve(tot, mom, Wf, fused=False), None, False
    sol = C.solve(tot, mom, Wf, fused=False)
    if sol["cond"] > 1e10 or sol["status"] != E.ECC_OK:
        return sol, None, True
    b_tot = C.sum_bound(t64, bnd, k) + (nt + 1) * C.U64 * np.abs(t64).sum(0)
    b_mom = 100 * C.U64 * np.abs(mp).sum(0)
    return sol, C.w_bound(tot, mom, Wf, b_tot, b_mom), True


def _e_cases():
    from oracle import oracle as O
    b = O.make_batch(3, 12)
    aug = np.zeros((12, 11), np.float32)
    aug[0] = [1, 1.1, 1.3, 0.9, 1.05, 1.15, 0.85, 0.7, 1.1, 0.95, 1.0]
    g1, g2 = E.prep(b["I_u8"], b["I_prime_u8"], aug)
    cases = [(g1[s], g2[s], np.eye(3, dtype=np.float32), "pairs[%d]" % s) for s in range(12)]
    ys, xs = np.mgrid[0:240, 0:320].astype(np.float64)
    img = 128 + 60 * np.sin(xs / 17.0) * np.cos(ys / 23.0) + 30 * np.sin((xs + ys) / 41.0)
    Wt = np.array([[1.0, 0.004, 1.6], [-0.003, 1.0, -1.2], [0.0, 0.0, 1.0]], np.float32)
    sm = (np.clip(img, 0, 255).astype(np.uint8), np.clip(E.warp_linear(img.astype(np.float32), np.linalg.inv(Wt)), 0, 255).astype(np.uint8))
    cases.append((sm[0], sm[1], np.eye(3, dtype=np.float32), "smooth"))
    for kind in K.KINDS:
        T, Im, Wf = K.case(kind, 240, 320, seed=4)
        cases.append((T, Im, Wf, kind))
    return cases


@pytest.mark.parametrize("kernel", KERNELS)
def test_one_iteration_against_the_float64_truth(kernel):
    """|W - W_fp64| after one iteration within the first-order propagation of the sums' bounds through the solve (x2) plus
    the float32 update rounding, per pair, at 240x320; statuses equal the truth's where it is not within its bound of a
    threshold."""
    _need_gpu()
    cases = _e_cases()
    T = np.stack([c[0] for c in cases]); Im = np.stack([c[1] for c in cases]); W0 = np.stack([c[2] for c in cases])
    out = run(kernel, T, Im, W0, 1)
    k = C.SPLIT_PX_PER_THREAD if kernel == "split" else C.one_cta_px_per_thread(240, 320)
    nt = layout(1, 240, 320)[1] if kernel == "split" else C.ONE_CTA_THREADS_Y
    worst, checked = 0.0, 0
    for s, (_, _, Wf, name) in enumerate(cases):
        tr = _truth(T[s], Im[s], Wf, k, nt)
        if tr is None:
            print("%s: a mean within 1e-12 of a float32 rounding boundary; skipped" % name)
            continue
        sol, wb, finite = tr
        if name in ("none", "flat"):
            assert out["status"][s] == sol["status"] == E.ECC_NAN, name
            continue
        if not finite:                                                   # den0: NaN Hessian; cv2 takes the same branch
            assert out["status"][s] == sol["status"], (name, out["status"][s], sol["status"])
            continue
        if sol["cond"] > 1e10:                                           # a Hessian of rank < 8 (a handful of pixels)
            print("%s: Hessian condition %.2e, W not compared" % (name, sol["cond"]))
            continue
        if abs(sol["lambda_d"]) > 1e-6 * (abs(sol["corr"]) + abs(sol["tpH"])):
            assert out["status"][s] == sol["status"], (name, out["status"][s], sol["status"], sol["lambda_d"])
        if wb is None or out["status"][s] != E.ECC_OK:
            continue
        d = np.abs(out["W"][s].astype(np.float64) - sol["W"].astype(np.float64))
        r = d / np.where(wb > 0, wb, 1)
        print("%s %s: worst |W - W_fp64| / bound %.3e (max |dW| %.3e)" % (kernel, name, r.max(), d.max()))
        assert np.all(d <= wb), (name, d, wb)
        worst = max(worst, float(r.max()))
        checked += 1
    assert checked >= 8
    _note("E %s W vs fp64 truth / propagated bound" % kernel, worst)


# ---- F. iteration state and stopping ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", KERNELS)
def test_iteration_state_and_stopping(kernel):
    """K = 5 iterations with eps = 0 equal five chained one-iteration runs bit for bit; with eps set to each observed
    |rho_i - rho_i-1| the count, status, W and rho follow the stopping rule on the kernel's own rho sequence;
    max_iters = 0 returns W_init, rho = -1 and 0 iterations."""
    _need_gpu()
    T, Im, Wf = K.case("perturbed", 240, 320, seed=6)
    T, Im, W0 = T[None], Im[None], Wf[None]
    chain_W, chain_rho, chain_st = [W0.reshape(9)], [-1.0], []
    for i in range(5):
        o = run(kernel, T, Im, chain_W[-1][None], 1)
        chain_W.append(o["W"][0]); chain_rho.append(o["rho"][0]); chain_st.append(o["status"][0])
    assert all(s == E.ECC_OK for s in chain_st)
    five = run(kernel, T, Im, W0, 5)
    assert five["iters"][0] == 5 and five["status"][0] == E.ECC_OK
    assert np.array_equal(five["W"][0], chain_W[5]) and five["rho"][0] == chain_rho[5]
    zero = run(kernel, T, Im, W0, 0)
    assert np.array_equal(zero["W"][0], W0.reshape(9)) and zero["rho"][0] == -1.0 and zero["iters"][0] == 0 and zero["status"][0] == 0
    deltas = [abs(chain_rho[i] - chain_rho[i - 1]) for i in range(2, 6)]
    for eps in sorted(set(deltas)):
        it, last, rho = 0, -eps, -1.0
        while it < 5 and abs(rho - last) >= eps:                     # the rule, on the kernel's own rho sequence
            it += 1
            last, rho = rho, chain_rho[it]
        o = run(kernel, T, Im, W0, 5, eps)
        assert (o["iters"][0], o["status"][0]) == (it, 0), (eps, o["iters"][0], it)
        assert np.array_equal(o["W"][0], chain_W[it]) and o["rho"][0] == chain_rho[it]
    print("%s: rho sequence %s, stops checked at %s" % (kernel, ["%.9f" % r for r in chain_rho[1:]], sorted(set(deltas))))
