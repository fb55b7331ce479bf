"""GPU tests of the real-data input pipeline and the real-data direct-method harness: each kernel equals its NumPy
restatement bit for bit, the device extended batch equals the host loader's in every key, the CNN's real test mode prints
the same metrics with either loader, and the harness's numbers are the library's."""
import os

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from oracle import jpeg as J  # noqa: E402
from oracle import real as R  # noqa: E402
from oracle import resize as Z  # noqa: E402

pytestmark = pytest.mark.gpu


def _bits(t):
    return np.asarray(t, np.float32).view(np.uint32)


# ---- kernels against the restatement ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("sh,sw,dh,dw", [(142, 190, 240, 320), (100, 130, 171, 250)])
def test_resize_area_up_u8_equals_the_oracle(sh, sw, dh, dw):
    from unsuperviseddeephomographyral2018_b200 import ops
    rng = np.random.default_rng(sh)
    src = rng.integers(0, 256, (3, sh, sw, 3)).astype(np.uint8)
    got = ops.resize_area_up_u8(torch.from_numpy(src).cuda(), dh, dw).cpu().numpy()
    for k in range(3):
        assert np.array_equal(got[k], Z.resize_area_up_u8(src[k], dh, dw)), k


@pytest.mark.parametrize("FH,FW,Hh,W", [(240, 320, 142, 190), (200, 300, 130, 170), (142, 190, 142, 190)])
@pytest.mark.parametrize("mode", ["train", "test"])
def test_real_prep_equals_the_oracle(FH, FW, Hh, W, mode):
    from unsuperviseddeephomographyral2018_b200 import ops
    rng = np.random.default_rng(FW)
    B = 3
    I, Ip = (rng.integers(0, 256, (B, FH, FW, 3)).astype(np.uint8) for _ in range(2))
    tables, _ = Z.draw_tables(rng, B, 0.7, mode)
    outs = ops.real_prep(torch.from_numpy(I).cuda(), torch.from_numpy(Ip).cuda(), torch.from_numpy(tables).cuda(), Hh, W)
    for t, out in enumerate(outs):
        got = out.cpu().numpy()
        for j in range(B):
            v = tables[j, t][(I if t % 2 == 0 else Ip)[j], np.arange(3)]
            ref = v if (FH, FW) == (Hh, W) else Z.resize_area_down_f32(v, Hh, W)
            assert np.array_equal(_bits(got[j]), _bits(ref)), (t, j)


def test_ecc_corr_h4p_equals_the_oracle():
    from unsuperviseddeephomographyral2018_b200 import _lib, ops
    rng = np.random.default_rng(3)
    B = 300
    W = np.tile(np.eye(3, dtype=np.float32), (B, 1, 1))
    W[:, :2, :2] += rng.normal(0, .02, (B, 2, 2)); W[:, :2, 2] += rng.normal(0, 10, (B, 2)); W[:, 2, :2] += rng.normal(0, 1e-4, (B, 2))
    c1 = rng.uniform(40, 600, (B, 8))
    gt = np.concatenate([c1, c1 + rng.normal(0, 8, (B, 8)) * (1 + 4 * (np.arange(B) % 3 == 0))[:, None]], 1).astype(np.float32)
    st = np.zeros(B, np.int32)
    W[0, 0, 2] = 400; W[1, 1, 2] = -300                                   # clamps
    st[2] = _lib.ECC_NAN; W[2] = np.nan; st[3] = _lib.ECC_NOCONV          # not found
    W[4] = [[1, 2, 0], [2, 4, 0], [0, 0, 1]]                               # singular, found
    W[5] = np.eye(3)
    pred, h, fail = ops.ecc_corr_h4p(torch.from_numpy(W).cuda(), torch.from_numpy(st).cuda(), torch.from_numpy(gt).cuda())
    rp, rh, rf = R.corr_h4p(W, st, gt)
    assert np.array_equal(fail.cpu().numpy(), rf) and set(rf.tolist()) == {0, 1, 2}
    assert np.array_equal(h.cpu().numpy().view(np.uint64), rh.view(np.uint64))
    assert np.array_equal(_bits(pred.cpu().numpy()), _bits(rp))


# ---- the loader ----------------------------------------------------------------------------------------------------------------
def _write_real_set(root, n=20, full=(240, 320), net=(142, 190), P=128, rho=4, seed=0, truncate=3):
    """The reference's real-data layout (I/, I_prime/, test_real.txt, test_pts1.txt, test_gt.txt with four clicked
    correspondences per pair): full-size and network-size JPEGs, gray files, restart markers, a progressive pair, a PNG
    pair and an odd-size pair (host fallback), and pair `truncate`'s I' cut in its entropy-coded data (device error)."""
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "I")); os.makedirs(os.path.join(root, "I_prime"))
    names, pts1, gt = [], [], []
    for i in range(n):
        name = "%06d.%s" % (i + 1, "png" if i == 5 else "jpg")
        for sub in ("I", "I_prime"):
            gray = (i + (sub == "I")) % 3 == 0
            hh, ww = (120, 160) if i == 7 else (full if i % 2 == 0 else net)
            img = J.textured(rng, hh, ww, 1 if gray else 3)
            prm = [cv2.IMWRITE_JPEG_QUALITY, 95] if i != 5 else []
            if i % 4 == 1:
                prm += [cv2.IMWRITE_JPEG_RST_INTERVAL, 3]
            if i == 11:
                prm += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
            path = os.path.join(root, sub, name)
            cv2.imwrite(path, img[..., 0] if gray else img[..., ::-1], prm)
            if i == truncate and sub == "I_prime":
                with open(path, "rb") as f:
                    b = f.read()
                with open(path, "wb") as f:
                    f.write(b[:len(b) * 2 // 3])
        names.append("%s %s" % (name, name))
        x0, y0 = rng.integers(rho, net[1] - rho - P + 1), rng.integers(rho, net[0] - rho - P + 1)
        pts1.append([x0, y0, x0 + P, y0, x0 + P, y0 + P, x0, y0 + P])
        c1 = rng.uniform(80, 560, 8)
        gt.append(np.concatenate([c1, c1 + rng.normal(0, 6, 8)]))
    with open(os.path.join(root, "test_real.txt"), "w") as f:
        f.write("\n".join(names) + "\n")
    np.savetxt(os.path.join(root, "test_pts1.txt"), np.array(pts1, np.float64))
    np.savetxt(os.path.join(root, "test_gt.txt"), np.array(gt, np.float64))


def _loader(root, mode, do_augment, B, img=(142, 190), full=(240, 320)):
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl
    prm = dl.extended_dataloader_params(data_path=str(root), filenames_file=os.path.join(root, "test_real.txt"),
                                        pts1_file=os.path.join(root, "test_pts1.txt"), gt_file=os.path.join(root, "test_gt.txt"),
                                        mode=mode, batch_size=B, img_h=img[0], img_w=img[1], patch_size=128, augment_list=["normalize"],
                                        do_augment=do_augment, full_img_h=full[0], full_img_w=full[1])
    return dl.Dataloader(prm, shuffle=True, seed=7, device="cuda")


def _copy(b):
    return {k: (v.clone() if isinstance(v, torch.Tensor) else (v.copy() if isinstance(v, np.ndarray) else v)) for k, v in b.items()}


@pytest.fixture(scope="module")
def real_set(tmp_path_factory):
    root = tmp_path_factory.mktemp("real")
    _write_real_set(root)
    return root


@pytest.mark.parametrize("B,mode,do_augment,nb", [(8, "train", 0.0, 4), (8, "train", 0.5, 4), (8, "train", 1.0, 4), (8, "test", 0.0, 4),
                                                  (8, "test", 0.5, 4), (8, "test", 1.0, 4), (1, "test", 0.5, 6), (128, "train", 0.5, 2),
                                                  (128, "test", 1.0, 2)])
def test_device_extended_batches_equal_the_host_loader(real_set, B, mode, do_augment, nb):
    dev, host = _loader(real_set, mode, do_augment, B), _loader(real_set, mode, do_augment, B)
    assert dev._extended_on_device()
    got = [_copy(dev.next_batch()) for _ in range(nb)]
    ref = [_copy(host._disk_batch_extended_host()) for _ in range(nb)]
    for k in range(nb):
        assert got[k].keys() == ref[k].keys()
        for key, v in ref[k].items():
            if isinstance(v, torch.Tensor):
                assert v.dtype == got[k][key].dtype and torch.equal(got[k][key], v), (k, key)
            elif isinstance(v, np.ndarray):
                assert v.dtype == got[k][key].dtype and np.array_equal(got[k][key], v), (k, key)
            else:
                assert v is None and got[k][key] is None, (k, key)
    st = dev.decode_stats
    assert st["device_images"] > 0
    if B * nb >= 20:                                                     # a whole epoch read: the fallbacks ran, the cut file failed on the device
        assert st["host_images"] > 0 and st["decode_errors"] >= 1


def test_full_size_equal_to_network_size(real_set):
    """Full size = network size: a table lookup, no resize; the other files (network-size and odd-size) take the host path."""
    dev = _loader(real_set, "test", 0.5, 8, img=(240, 320), full=(240, 320))
    host = _loader(real_set, "test", 0.5, 8, img=(240, 320), full=(240, 320))
    for _ in range(3):
        a, b = _copy(dev.next_batch()), _copy(host._disk_batch_extended_host())
        for key in ("I1", "I2", "I1_aug", "I2_aug", "I_aug", "I_prime_aug", "pts1", "patch_indices", "I_u8", "I_prime_u8", "aug"):
            assert torch.equal(a[key], b[key]), key
        assert np.array_equal(a["full_I"], b["full_I"]) and np.array_equal(a["gt_corr"], b["gt_corr"])


def test_unrestated_geometry_takes_the_host_path(real_set, monkeypatch):
    """An fp32 upscale (full size below the network size) is not restated: every batch runs the host code."""
    dev = _loader(real_set, "test", 0.5, 4, img=(142, 190), full=(120, 160))
    assert not dev._extended_on_device()
    calls = []
    real = type(dev)._disk_batch_extended_host
    monkeypatch.setattr(type(dev), "_disk_batch_extended_host", lambda self: calls.append(1) or real(self))
    b = dev.next_batch()
    assert calls and b["I_aug"].shape == (4, 142, 190, 3) and b["I_u8"].shape == (4, 120, 160, 3)


# ---- the CLIs -----------------------------------------------------------------------------------------------------------------
def _run_cli(script, argv, capsys, monkeypatch, host):
    import importlib
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    monkeypatch.syspath_prepend(root)
    mod = importlib.import_module(script)
    from unsuperviseddeephomographyral2018_b200 import dataloader
    with monkeypatch.context() as m:
        if host:
            m.setattr(dataloader.Dataloader, "_extended_on_device", lambda self: False)
        capsys.readouterr()
        rc = mod.main(argv)
        out = capsys.readouterr().out
    assert rc in (0, None), out[-2000:]
    sys.stdout.flush()
    return out


def test_cnn_real_test_mode_gives_the_same_metrics_with_either_loader(real_set, tmp_path, monkeypatch, capsys):
    outs = []
    for host in (False, True):
        argv = ["--mode", "test", "--data_path", str(real_set) + "/", "--batch_size", "8", "--num_gpus", "1", "--numeric", "bf16x3",
                "--do_augment", "0.5", "--load_model_dir", str(tmp_path / "m"), "--save_model_dir", str(tmp_path / "s"),
                "--log_dir", str(tmp_path / "l"), "--results_dir", str(tmp_path / "r")]
        lines = _run_cli("homography_CNN_real", argv, capsys, monkeypatch, host).splitlines()
        i = next(k for k, ln in enumerate(lines) if ln.startswith("|Steps"))
        outs.append(lines[i:i + 4])
    assert outs[0] == outs[1]
    assert len(outs[0][1].split()) == 4


def _results(log_dir):
    (path,) = [os.path.join(d, f) for d, _, fs in os.walk(log_dir) for f in fs if f == "results.txt"]
    with open(path) as f:
        return f.read().split()


def test_real_harness_numbers_are_the_library_numbers(real_set, tmp_path, monkeypatch, capsys):
    from unsuperviseddeephomographyral2018_b200 import ops
    res = {}
    for method in ("direct", "identity"):
        argv = ["--method", method, "--data_path", str(real_set) + "/", "--batch_size", "8", "--num_iterations", "20",
                "--log_dir", str(tmp_path / ("l" + method)), "--results_dir", str(tmp_path / ("r" + method))]
        out = _run_cli("homography_conventional_real", argv, capsys, monkeypatch, host=False)
        import homography_conventional_real as M
        assert "===> Percentile Values: (20, 50, 80, 100):" in out
        res[method] = _results(tmp_path / ("l" + method))
        args = M.resolve_paths(M.build_parser().parse_args(argv))
        loader = M.make_loader(args, 8)
        loader.shuffle = False
        h, f = [], []
        for _ in range(3):                                               # 20 pairs in batches of 8
            b = loader.next_batch()
            gt = torch.from_numpy(b["gt_corr"]).cuda()
            if method == "direct":
                g1, g2 = ops.ecc_prep_u8(b["I_u8"], b["I_prime_u8"], b["aug"])
                W, _, _, st = ops.find_homography_ecc(g1, g2, None, 20, 1e-10)
            else:
                W = torch.eye(3, device="cuda").repeat(8, 1, 1).contiguous(); st = torch.zeros(8, device="cuda", dtype=torch.int32)
            _, hh, ff = ops.ecc_corr_h4p(W, st, gt)
            h += hh.cpu().tolist(); f += ff.cpu().tolist()
            if method == "identity":
                c = b["gt_corr"] / np.float32(2)
                ident = np.sqrt(np.mean(np.square(c[:, :8] - c[:, 8:]), axis=1, dtype=np.float64))
                assert np.allclose(hh.cpu().numpy(), ident, rtol=1e-6, atol=0) and not ff.cpu().numpy().any()
        line = M.summarise(h, int(np.sum(np.asarray(f) != 0)), 0.0, len(h))
        assert res[method][:4] == ["%.5f" % v for v in line[:4]], (method, res[method], line)
    assert res["identity"][3] == "0.00000"


def test_real_harness_direct_beats_identity_on_synthetic_pairs(tmp_path, monkeypatch, capsys):
    res = {}
    for method in ("direct", "identity"):
        argv = ["--method", method, "--synthetic", "64", "--batch_size", "64", "--do_augment", "0",
                "--log_dir", str(tmp_path / ("l" + method)), "--results_dir", str(tmp_path / ("r" + method))]
        _run_cli("homography_conventional_real", argv, capsys, monkeypatch, host=False)
        res[method] = [float(v) for v in _results(tmp_path / ("l" + method))]
    assert res["identity"][3] == 0.0
    assert res["direct"][1] < res["identity"][1], res
