"""GPU tests of the dataset generator: udh_gen_warp_u8 equals the reference's numpy_transformer (gen_golden.npz) and the
NumPy restatement on random theta; gen_synthetic_data.py --seed s writes a directory byte-identical to the host
generator's (train with colour, train with --color false, test); the CNN CLI's test mode runs on the generated set with
every file decoded on the device."""
import os

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from oracle import gen_data as OG  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _theta(Hi, h, w):
    M = np.array([[w / 2.0, 0, w / 2.0], [0, h / 2.0, h / 2.0], [0, 0, 1.]]).astype(np.float32)
    return np.dot(np.dot(np.linalg.inv(M), np.linalg.inv(Hi)), M)


def test_device_warp_equals_the_reference_golden():
    from unsuperviseddeephomographyral2018_b200 import ops
    g = np.load(os.path.join(ROOT, "tests", "golden", "gen_golden.npz"))
    th = np.stack([_theta(Hi, 240, 320) for Hi in g["H_inverse"]])
    gray, warped, warped_gray = ops.gen_warp_u8(torch.from_numpy(g["bgr"]).cuda(), torch.from_numpy(th).cuda())
    assert np.array_equal(gray.cpu().numpy(), g["gray"])
    assert np.array_equal(warped.cpu().numpy(), g["warped"])
    assert np.array_equal(warped_gray.cpu().numpy(), g["warped_gray"])


@pytest.mark.parametrize("h,w", [(240, 320), (37, 53), (1, 7)])
def test_device_warp_equals_the_oracle_on_random_theta(h, w):
    from unsuperviseddeephomographyral2018_b200 import ops
    rng = np.random.default_rng(h * 100 + w)
    n = 24
    img = rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    th = np.eye(3)[None] + rng.standard_normal((n, 3, 3)) * np.array([[0.3, 0.3, 0.5], [0.3, 0.3, 0.5], [0.2, 0.2, 0.3]])
    th[-1] = [[3.0, 0.1, 4.0], [0.2, 2.5, -5.0], [0.9, -0.8, 0.01]]       # far outside the image, weights far outside [0, 1]
    gray, warped, warped_gray = (t.cpu().numpy() for t in ops.gen_warp_u8(torch.from_numpy(img).cuda(), torch.from_numpy(th).cuda()))
    for k in range(n):
        g = OG.gray(img[k])
        assert np.array_equal(gray[k], g), k
        assert np.array_equal(warped[k], OG.warp(img[k], th[k])), k
        assert np.array_equal(warped_gray[k], OG.warp(g, th[k])), k


def _tree(root):
    out = {}
    for d, _, fs in os.walk(root):
        for f in fs:
            p = os.path.join(d, f)
            with open(p, "rb") as fh:
                out[os.path.relpath(p, root)] = fh.read()
    return out


@pytest.mark.parametrize("mode,color", [("train", True), ("train", False), ("test", True)])
def test_device_generator_directory_is_byte_identical_to_the_host_generator(tmp_path, mode, color):
    from test_gen_data_oracle import gen_args, write_raw_set
    from unsuperviseddeephomographyral2018_b200 import gen_data as G
    write_raw_set(tmp_path / "raw")
    trees = []
    for side in ("device", "host"):
        base = tmp_path / side
        os.makedirs(base, exist_ok=True)
        os.symlink(tmp_path / "raw", base / "raw")
        args = gen_args(base, mode, color=color, num_data=11, test_num_data=7)
        if side == "device":
            argv = ["--mode", mode, "--color", "true" if color else "false", "--raw_data_path", str(base / "raw"),
                    "--test_raw_data_path", str(base / "raw"), "--data_path", str(base / "data") + "/", "--num_data", "11",
                    "--test_num_data", "7", "--seed", "9"]
            G.main(argv)
        else:
            G.generate(args, OG.HostBackend(), seed=9)
        trees.append(_tree(base / "data"))
    dev, host = trees
    assert sorted(dev) == sorted(host) and len(dev) >= 2 * 7 + 3
    for name in host:
        assert dev[name] == host[name], name
    sample = cv2.imread(str(tmp_path / "device" / "data" / "I" / sorted(n for n in dev if n.startswith("I/"))[0][2:]),
                        cv2.IMREAD_UNCHANGED)
    assert sample.shape == ((240, 320) if (mode == "train" and not color) else (240, 320, 3))


def test_cnn_test_mode_runs_on_a_generated_set_with_every_file_decoded_on_the_device(tmp_path, monkeypatch, capsys):
    import importlib
    from test_gen_data_oracle import write_raw_set
    from unsuperviseddeephomographyral2018_b200 import dataloader, gen_data as G
    write_raw_set(tmp_path / "raw")
    data = str(tmp_path / "data") + "/"
    G.main(["--mode", "test", "--test_raw_data_path", str(tmp_path / "raw"), "--data_path", data, "--num_data", "0",
            "--test_num_data", "12", "--seed", "4"])
    prm = dataloader.dataloader_params(data_path=data, filenames_file=data + "test_synthetic.txt", pts1_file=data + "test_pts1.txt",
                                       gt_file=data + "test_gt.txt", mode="test", batch_size=4, img_h=240, img_w=320, patch_size=128,
                                       augment_list=["normalize"], do_augment=0.0)
    dl = dataloader.Dataloader(prm, shuffle=False, seed=0)
    for _ in range(3):
        dl.next_batch()
    torch.cuda.synchronize()
    st = dl.decode_stats
    assert st["device_images"] >= 24 and st["host_images"] == 0 and st["decode_errors"] == 0, st
    monkeypatch.syspath_prepend(ROOT)
    mod = importlib.import_module("homography_CNN_synthetic")
    argv = ["--mode", "test", "--data_path", data, "--batch_size", "4", "--num_gpus", "1", "--numeric", "bf16x3",
            "--model_dir", str(tmp_path / "m"), "--log_dir", str(tmp_path / "l"), "--results_dir", str(tmp_path / "r")]
    capsys.readouterr()
    rc = mod.main(argv)
    out = capsys.readouterr().out
    assert rc in (0, None), out[-2000:]
    assert any(ln.startswith("|Steps") for ln in out.splitlines()), out[-2000:]
