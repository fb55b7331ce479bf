"""CPU tests of the real-data loader's restatement (oracle/resize.py), the real harness's metric (oracle/real.py) and the
real-data direct-method CLI's arguments and output files."""
import os
import pickle

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import real as R  # noqa: E402
from oracle import resize as Z  # noqa: E402

MEAN = np.array([118.93, 113.97, 102.60], np.float32)
STD = np.array([69.85, 68.81, 72.45], np.float32)


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


@pytest.mark.parametrize("sh,sw,dh,dw", [(240, 320, 142, 190), (200, 300, 130, 170), (240, 320, 120, 190), (99, 77, 40, 50)])
def test_area_downscale_f32_is_cv2(sh, sw, dh, dw):
    rng = np.random.default_rng(sh + dw)
    for _ in range(2):
        u8 = rng.integers(0, 256, (sh, sw, 3)).astype(np.float32)
        x = (np.clip(u8 ** np.float32(rng.uniform(0.8, 1.2)) * np.float32(1.3), 0, 255) - MEAN) / STD
        assert _bits_equal(Z.resize_area_down_f32(x, dh, dw), cv2.resize(x, (dw, dh), interpolation=cv2.INTER_AREA))


@pytest.mark.parametrize("sh,sw,dh,dw", [(142, 190, 240, 320), (100, 130, 171, 250), (60, 70, 97, 101)])
def test_area_upscale_u8_is_cv2(sh, sw, dh, dw):
    rng = np.random.default_rng(sh)
    for _ in range(3):
        im = rng.integers(0, 256, (sh, sw, 3)).astype(np.uint8)
        assert np.array_equal(Z.resize_area_up_u8(im, dh, dw), cv2.resize(im, (dw, dh), interpolation=cv2.INTER_AREA))


def test_generic_area_path_excludes_integer_ratios_and_upscales():
    assert Z.area_is_generic(240, 320, 142, 190) and Z.area_is_generic(240, 320, 120, 190)
    assert not Z.area_is_generic(240, 320, 120, 160) and not Z.area_is_generic(142, 190, 240, 320)


def test_value_tables_reproduce_the_host_expression():
    rng = np.random.default_rng(1)
    for _ in range(10):
        u8 = rng.integers(0, 256, (60, 80, 3)).astype(np.uint8)
        a = u8.astype(np.float32)
        g, br, c = rng.uniform(0.8, 1.2), rng.uniform(0.5, 2.0), rng.uniform(0.8, 1.2, size=3).astype(np.float32)
        host = (np.clip(a ** np.float32(g) * np.float32(br) * c, 0, 255) - MEAN) / STD
        assert _bits_equal(Z.value_table(g, br, c)[u8, np.arange(3)], host)
        assert _bits_equal(Z.value_table()[u8, np.arange(3)], (a - MEAN) / STD)


def test_library_tables_equal_the_restatement():
    from unsuperviseddeephomographyral2018_b200 import ops
    tab, max_rows = ops.area_table(240, 320, 142, 190)
    nx, ny = tab[0], tab[1]
    xo, xs = tab[2:2 + 191], tab[2 + 191:2 + 191 + nx]
    xw = tab[2 + 191 + nx:2 + 191 + 2 * nx].view(np.float32)
    ref = Z.area_tab(320, 190)
    assert nx == len(ref) and ny == len(Z.area_tab(240, 142)) and max_rows == 3
    assert [(d, s, w) for d, s, w in ref] == [(int(np.searchsorted(xo, k, 'right') - 1), int(xs[k]), xw[k]) for k in range(nx)]
    up = ops.linear_area_table(142, 190, 240, 320)
    sx, ax = Z.linear_area_coefs(190, 320)
    sy, ay = Z.linear_area_coefs(142, 240)
    assert np.array_equal(up, np.concatenate([sx, ax[:, 0], ax[:, 1], sy, ay[:, 0], ay[:, 1]]))


def _write_real_set(root, n=6, seed=0, full=(240, 320), net=(142, 190), P=128, rho=4):
    rng = np.random.default_rng(seed)
    for sub in ("I", "I_prime"):
        os.makedirs(os.path.join(root, sub), exist_ok=True)
    names, pts1, gt = [], [], []
    for i in range(n):
        name = "%03d.png" % i
        h, w = full if i % 2 == 0 else net
        for sub in ("I", "I_prime"):
            cv2.imwrite(os.path.join(root, sub, name), rng.integers(0, 256, (h, w, 3)).astype(np.uint8))
        names.append("%s %s" % (name, name))
        x0, y0 = rng.integers(rho, net[1] - rho - P), rng.integers(rho, net[0] - rho - P)
        pts1.append([x0, y0, x0 + P, y0, x0 + P, y0 + P, x0, y0 + P])
        gt.append(rng.uniform(20, 460, 16))
    with open(os.path.join(root, "list.txt"), "w") as f:
        f.write("\n".join(names) + "\n")
    np.savetxt(os.path.join(root, "pts1.txt"), np.array(pts1, np.float64))
    np.savetxt(os.path.join(root, "gt.txt"), np.array(gt, np.float64))


def _extended_loader(root, mode, do_augment, B, seed=5):
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl
    prm = dl.extended_dataloader_params(data_path=str(root), filenames_file=os.path.join(root, "list.txt"),
                                        pts1_file=os.path.join(root, "pts1.txt"), gt_file=os.path.join(root, "gt.txt"), mode=mode,
                                        batch_size=B, img_h=142, img_w=190, patch_size=128, augment_list=["normalize"],
                                        do_augment=do_augment, full_img_h=240, full_img_w=320)
    return dl.Dataloader(prm, shuffle=True, seed=seed, device="cpu")


@pytest.mark.parametrize("mode", ["train", "test"])
@pytest.mark.parametrize("do_augment", [0.0, 0.5, 1.0])
def test_table_builder_draws_what_the_host_loader_draws(tmp_path, mode, do_augment):
    """The oracle's builder and the loader's device-path draw consume the host path's RNG numbers in its order, and their
    tables give the host batch's fp32 images through the restated resize."""
    _write_real_set(tmp_path)
    host, dev = _extended_loader(tmp_path, mode, do_augment, 4), _extended_loader(tmp_path, mode, do_augment, 4)
    for step in range(3):                                                 # 12 pairs of a 6-pair set: two epoch wraps
        idx, tables, aug = dev._draw_batch_extended()
        b = host._disk_batch_extended_host()
        assert host._rng.bit_generator.state == dev._rng.bit_generator.state
        assert np.array_equal(b["aug"].numpy(), aug)
        I_u8, Ip_u8 = b["I_u8"].numpy(), b["I_prime_u8"].numpy()
        assert np.array_equal(I_u8, b["full_I"]) and np.array_equal(Ip_u8, b["full_I_prime"])
        for j in range(4):
            for k, src, key in ((2, I_u8, "I_aug"), (3, Ip_u8, "I_prime_aug")):
                ref = Z.resize_area_down_f32(tables[j, k][src[j], np.arange(3)], 142, 190)
                assert _bits_equal(ref, b[key].numpy()[j]), (step, j, key)


def test_oracle_table_builder_matches_the_loader_draw():
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl
    for mode in ("train", "test"):
        for do_augment in (0.0, 0.5, 1.0):
            prm = dl.extended_dataloader_params(data_path="", filenames_file="", pts1_file="", gt_file="", mode=mode, batch_size=16,
                                                img_h=142, img_w=190, patch_size=128, augment_list=["normalize"], do_augment=do_augment,
                                                full_img_h=240, full_img_w=320)
            loader = dl.Dataloader(prm, synthetic_pairs=1, seed=11, device="cpu")
            loader.num_samples, loader._order, loader._cursor = 16, np.arange(16), 16
            loader.shuffle = False
            rng = np.random.default_rng(11)
            _, tables, aug = loader._draw_batch_extended()
            ref_tables, ref_aug = Z.draw_tables(rng, 16, do_augment, mode)
            assert _bits_equal(tables, ref_tables) and _bits_equal(aug, ref_aug)
            assert rng.bit_generator.state == loader._rng.bit_generator.state
            if do_augment == 0.0:
                assert not aug.any()
            if do_augment == 1.0:
                assert aug[:, 0].all() and (mode == "test") != np.array_equal(aug[:, 1:6], aug[:, 6:11])


# ---- the metric -----------------------------------------------------------------------------------------------------------
def _reference_loop(W, not_found, gt):
    """homography_conventional_real.py:213-246 with direct_homography.py:42-57 (return_h_inv=False), transcribed."""
    out = []
    for i in range(len(gt)):
        corr1 = gt[i, 0:8].reshape([4, 2]) / 2
        corr2 = gt[i, 8:16].reshape([4, 2]) / 2
        if not_found[i]:
            pred_h4p = np.zeros([1, 4, 2])
        else:
            corners = np.float32(corr1).reshape(1, 4, 2)
            pred_h4p = cv2.perspectiveTransform(corners, W[i]) - corners
        pred_h4p[np.where(pred_h4p >= 80)] = 80
        pred_h4p[np.where(pred_h4p <= -80)] = -80
        pred_corr2 = pred_h4p[0] + corr1
        h = np.sqrt(np.mean(np.square(pred_corr2 - corr2)))
        fail = 0
        if not_found[i]:
            fail = 1
        else:
            ident = np.sqrt(np.mean(np.square(corr1 - corr2)))
            if ident < h:
                fail, h = 2, ident
        out.append((pred_h4p.reshape(8).astype(np.float32), float(h), fail))
    return out


def _hand_made_cases():
    rng = np.random.default_rng(3)
    Ws, st, gts = [], [], []
    for k in range(40):
        c1 = rng.uniform(40, 600, (4, 2))
        W = np.eye(3) + np.array([[rng.normal(0, .02), rng.normal(0, .02), rng.normal(0, 8)],
                                  [rng.normal(0, .02), rng.normal(0, .02), rng.normal(0, 8)],
                                  [rng.normal(0, 1e-4), rng.normal(0, 1e-4), 0]])
        c2 = (c1 + rng.normal(0, 6, (4, 2))) if k % 3 else c1 + rng.normal(0, 40, (4, 2))
        Ws.append(W); st.append(0); gts.append(np.concatenate([c1.reshape(-1), c2.reshape(-1)]))
    Ws[0] = np.eye(3); Ws[0][0, 2] = 300.0                               # clamp at +80
    Ws[1] = np.eye(3); Ws[1][1, 2] = -250.0                              # clamp at -80
    Ws[2] = np.full((3, 3), np.nan); st[2] = 1                           # ECC raised on NaN: fail 1
    Ws[3] = np.zeros((3, 3)); st[3] = 2                                  # singular / no convergence: fail 1
    Ws[4] = np.array([[1, 2, 0], [2, 4, 0], [0, 0, 1.0]])                # singular but found: scored as it is
    Ws[5] = np.array([[1, 0, 0], [0, 1, 0], [-1, 0, 0.0]])               # w <= FLT_EPSILON at x = 0? points map to 0
    Ws[6] = np.eye(3)                                                    # identity: h = identity error, no failure
    return np.array(Ws, np.float32), np.array(st, np.int32), np.array(gts, np.float32)


def test_metric_restatement_matches_the_reference_loop():
    W, st, gt = _hand_made_cases()
    pred, h, fail = R.corr_h4p(W, st, gt)
    ref = _reference_loop(W, st != 0, gt)
    for b, (p, hv, f) in enumerate(ref):
        assert fail[b] == f, b
        assert h[b] == hv, (b, h[b], hv)
        if not st[b]:
            assert _bits_equal(pred[b], p), b
    assert set(fail.tolist()) == {0, 1, 2}
    assert pred[0].max() == 80 and pred[1].min() == -80
    assert fail[6] == 0 and h[6] == float(np.sqrt(np.mean(np.square(gt[6, :8] / 2 - gt[6, 8:] / 2))))


# ---- the CLI ----------------------------------------------------------------------------------------------------------------
def _cli():
    import importlib
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    return importlib.import_module("homography_conventional_real")


def test_cli_defaults_and_directories():
    m = _cli()
    a = m.resolve_paths(m.build_parser().parse_args(["--method", "direct", "--data_path", "/d/", "--log_dir", "/l", "--results_dir", "/r"]))
    assert (a.num_iterations, a.img_h, a.img_w, a.full_img_h, a.full_img_w, a.patch_size, m.RHO) == (100, 142, 190, 240, 320, 128, 24)
    assert (a.mode, a.do_augment, a.batch_size, a.num_features, a.max_epoches, a.artifact_mode) == ('test', 0.5, 128, 8, 1, 'None')
    assert a.log_dir == "/l/direct/_normalize/RHO_24_maxfeat_8_doaugment_0.5/test/"
    assert a.results_dir == "/r/direct/_normalize/RHO_24_maxfeat_8_doaugment_0.5/test/"
    assert (a.test_filenames_file, a.test_pts1_file, a.test_gt_file) == ("/d/test_real.txt", "/d/test_pts1.txt", "/d/test_gt.txt")
    assert m.build_parser().parse_args([]).method == 'SIFT'


@pytest.mark.parametrize("argv", [["--method", "SIFT"], ["--method", "ORB"], ["--method", "direct", "--mode", "train"]])
def test_cli_refuses_what_is_not_built(argv, tmp_path):
    m = _cli()
    assert m.main(argv + ["--log_dir", str(tmp_path / "l"), "--results_dir", str(tmp_path / "r")]) == 2


def test_cli_output_files(tmp_path):
    m = _cli()
    a = m.resolve_paths(m.build_parser().parse_args(["--method", "identity", "--log_dir", str(tmp_path / "l"),
                                                     "--results_dir", str(tmp_path / "r")]))
    os.makedirs(a.log_dir); os.makedirs(a.results_dir)
    h = [1.5, 2.25, np.float32(3.125)]
    line = m.summarise(h, 1, 0.3, 3)
    m.write_pickle(a, h)
    m.write_results_txt(a, line)
    with open(os.path.join(a.results_dir, "h_losses.pkl"), "rb") as f:
        d = pickle.load(f)
    assert d == {'method': 'identity', 'h_losses': [1.5, 2.25, 3.125], 'h_loss_mu': float(np.mean(h)), 'h_loss_std': float(np.std(h))}
    with open(os.path.join(a.log_dir, "results.txt")) as f:
        assert f.read() == "3.00000 %.5f %.5f 0.33333 0.10000\n" % (np.mean(h), np.std(h))
    tops = m.find_percentile(list(range(10)))
    assert tops == [[1.0, float(np.std([0, 1, 2]))], [4.0, float(np.std([3, 4, 5]))], [7.5, float(np.std([6, 7, 8, 9]))]]
