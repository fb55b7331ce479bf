"""GPU tests of the direct-method baseline (csrc/ecc.cu) against the NumPy restatement oracle/ecc.py and the stored
OpenCV outcomes tests/golden/ecc_golden.npz."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import ecc as E
from oracle import oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AUG0 = [1, 1.1, 1.3, 0.9, 1.05, 1.15, 0.85, 0.7, 1.1, 0.95, 1.0]


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _pairs():
    b = O.make_batch(3, 12)
    aug = np.zeros((12, 11), np.float32); aug[0] = AUG0
    return b, aug


def _smooth_pair():
    ys, xs = np.mgrid[0:240, 0:320].astype(np.float64)
    img = 128 + 60 * np.sin(xs / 17.0) * np.cos(ys / 23.0) + 30 * np.sin((xs + ys) / 41.0)
    Wt = np.array([[1.0, 0.004, 1.6], [-0.003, 1.0, -1.2], [0.0, 0.0, 1.0]], np.float32)
    return np.clip(img, 0, 255).astype(np.uint8), np.clip(E.warp_linear(img.astype(np.float32), np.linalg.inv(Wt)), 0, 255).astype(np.uint8)


def _corner_dist(Wa, Wb, H=240, Wd=320):
    c = np.array([[0, 0, 1], [Wd - 1, 0, 1], [Wd - 1, H - 1, 1], [0, H - 1, 1]], np.float64).T
    pa = np.asarray(Wa, np.float64).reshape(3, 3) @ c; pb = np.asarray(Wb, np.float64).reshape(3, 3) @ c
    return float(np.abs(pa[:2] / pa[2] - pb[:2] / pb[2]).max())


def _run(g1, g2, k):
    from unsuperviseddeephomographyral2018_b200 import ops
    W, rho, it, st = ops.find_homography_ecc(torch.as_tensor(g1).cuda(), torch.as_tensor(g2).cuda(), None, k)
    torch.cuda.synchronize()
    return W.cpu().numpy(), rho.cpu().numpy(), it.cpu().numpy(), st.cpu().numpy()


def test_prep_kernel_is_bit_identical_to_the_oracle():
    _need_gpu()
    from unsuperviseddeephomographyral2018_b200 import ops
    b, aug = _pairs()
    aug[3] = [1, 0.85, 0.6, 1.2, 0.8, 1.0, 1.2, 1.9, 0.9, 1.1, 0.85]      # disjoint draw
    g1, g2 = ops.ecc_prep_u8(torch.as_tensor(b["I_u8"]).cuda(), torch.as_tensor(b["I_prime_u8"]).cuda(), torch.as_tensor(aug).cuda())
    r1, r2 = E.prep(b["I_u8"], b["I_prime_u8"], aug)
    assert np.array_equal(g1.cpu().numpy(), r1) and np.array_equal(g2.cpu().numpy(), r2)
    n1, _ = ops.ecc_prep_u8(torch.as_tensor(b["I_u8"]).cuda(), torch.as_tensor(b["I_prime_u8"]).cuda(), None)
    assert np.array_equal(n1.cpu().numpy(), E.prep(b["I_u8"], b["I_prime_u8"], None)[0])


def test_iterations_match_the_oracle_and_opencv_outcomes():
    """After 1 iteration W sends the image corners within 2e-2 px of the oracle's fp64 restatement (measured on an H100:
    5.7e-3 px, on a pair with rho = 0.003 whose Hessian amplifies the fp32 per-thread partial sums; cv2 and the oracle
    differ by 0.05 px there); on the converging pair within 1e-2 px after 8.  Status and iteration count match the oracle and cv2's stored outcome on every pair (none of
    them is decided by a quantity within 1e-4 relative of its threshold: test_ecc_oracle.py)."""
    _need_gpu()
    b, aug = _pairs()
    g1, g2 = E.prep(b["I_u8"], b["I_prime_u8"], aug)
    z = np.load(os.path.join(ROOT, "tests", "golden", "ecc_golden.npz"))
    W1, _, it1, st1 = _run(g1, g2, 1)
    W8, rho8, it8, st8 = _run(g1, g2, 8)
    worst1 = 0.0
    for s in range(12):
        o1 = E.ecc(g1[s], g2[s], max_iters=1)
        o8 = E.ecc(g1[s], g2[s], max_iters=8)
        assert (st1[s], it1[s]) == (o1["status"], o1["iters"]), s
        assert (st8[s], it8[s]) == (o8["status"], o8["iters"]), s
        assert st8[s] == int(z["status"][s]), s
        if st1[s] == E.ECC_OK:
            worst1 = max(worst1, _corner_dist(W1[s], o1["W"]))
    print("1 iteration: worst corner distance to the oracle %.3e px" % worst1)
    assert worst1 < 2e-2
    t, im = _smooth_pair()
    W, rho, it, st = _run(t[None], im[None], 8)
    o = E.ecc(t, im, max_iters=8)
    d = _corner_dist(W[0], o["W"])
    print("converging pair, 8 iterations: corner distance %.3e px, rho %.6f (oracle %.6f)" % (d, rho[0], o["rho"]))
    assert st[0] == E.ECC_OK and it[0] == 8 and d < 1e-2 and abs(rho[0] - o["rho"]) < 1e-5


def test_runs_and_batch_positions_are_bit_identical():
    _need_gpu()
    b, aug = _pairs()
    g1, g2 = E.prep(b["I_u8"], b["I_prime_u8"], aug)
    t, im = _smooth_pair()
    B = 64
    T = np.concatenate([np.tile(g1, (5, 1, 1)), t[None].repeat(4, 0)])[:B]
    I = np.concatenate([np.tile(g2, (5, 1, 1)), im[None].repeat(4, 0)])[:B]
    a = _run(T, I, 8); c = _run(T, I, 8)
    for x, y in zip(a, c):
        assert np.array_equal(x, y, equal_nan=True)
    for s in (0, 4, 61):
        one = _run(T[s:s + 1], I[s:s + 1], 8)
        for x, y in zip(one, a):
            assert np.array_equal(x[0], y[s], equal_nan=True)


def test_h4p_kernel_matches_the_oracle():
    _need_gpu()
    from unsuperviseddeephomographyral2018_b200 import ops
    b, aug = _pairs()
    g1, g2 = E.prep(b["I_u8"], b["I_prime_u8"], aug)
    W, _, _, st = _run(g1, g2, 8)
    W[0] = np.array([[1, 0, -3.0], [0, 1, 2.0], [0, 0, 1]], np.float32); st[0] = E.ECC_OK   # a known shift: fail case 2
    pred, h, fail = ops.ecc_h4p(torch.as_tensor(W).cuda(), torch.as_tensor(st).cuda(), b["pts1"].cuda(), b["gt"].cuda(), 45.0)
    for s in range(12):
        rp, rh, rf = E.h4p(W[s], int(st[s]), b["pts1"][s].numpy(), b["gt"][s].numpy())
        assert np.array_equal(pred[s].cpu().numpy(), rp), s
        assert int(fail[s]) == rf and float(h[s]) == pytest.approx(rh, rel=1e-6), s


def test_cli_direct_writes_results_matching_the_library(tmp_path):
    _need_gpu()
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "homography_conventional_synthetic.py"), "--method", "direct", "--synthetic", "64",
                        "--batch_size", "64", "--log_dir", str(tmp_path) + "/"], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert re.search(r"H_loss: .* \+/- ", r.stdout) and "Percentile Values" in r.stdout and "batched" in r.stdout
    res = os.path.join(str(tmp_path), "direct", "_normalize", "RHO_45_maxfeat_8_doaugment_0.5", "test", "results.txt")
    got = np.loadtxt(res)
    # recompute from the library's per-sample outputs on the same batch
    sys.path.insert(0, ROOT)
    import homography_conventional_synthetic as C
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl
    dp = dl.dataloader_params(data_path="", filenames_file="", pts1_file="", gt_file="", mode='test', batch_size=64, img_h=240, img_w=320,
                              patch_size=128, augment_list=['normalize'], do_augment=0.5)
    batch = dl.Dataloader(dp, shuffle=False, synthetic_pairs=64, seed=0, device="cuda").next_batch()
    h, f, _ = C.run_batch('direct', batch, 8, 45)
    line = C.summarise(h, f, 0.0, 64)
    assert got[0] == 64 and np.allclose(got[1:4], np.round(line[1:4], 5), atol=1.5e-5)
    r2 = subprocess.run([sys.executable, os.path.join(ROOT, "homography_conventional_synthetic.py"), "--method", "SIFT", "--synthetic", "4",
                         "--log_dir", str(tmp_path) + "/"], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert r2.returncode != 0 and "not built" in r2.stderr
