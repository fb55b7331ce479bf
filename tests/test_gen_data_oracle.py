"""CPU tests of the dataset generator: the warp restatement equals the reference's numpy_transformer (gen_golden.npz) bit
for bit, the gray rule equals cv2, and the host generator's draws, names, text files and cutoffs equal a transcription of
the reference's homographyGeneration loop, in a layout read_img_and_gt parses."""
import os

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import gen_data as OG  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _theta(Hi, h, w):
    M = np.array([[w / 2.0, 0, w / 2.0], [0, h / 2.0, h / 2.0], [0, 0, 1.]]).astype(np.float32)
    return np.dot(np.dot(np.linalg.inv(M), np.linalg.inv(Hi)), M)


def test_warp_oracle_equals_the_reference_golden():
    g = np.load(os.path.join(ROOT, "tests", "golden", "gen_golden.npz"))
    for k in range(len(g["bgr"])):
        th = _theta(g["H_inverse"][k], 240, 320)
        assert np.array_equal(OG.gray(g["bgr"][k]), g["gray"][k])
        assert np.array_equal(OG.warp(g["bgr"][k], th), g["warped"][k])
        assert np.array_equal(OG.warp(g["gray"][k], th), g["warped_gray"][k])
        assert (g["warped_gray"][k] == 0).sum() > 1000                 # out-of-image pixels are part of the comparison


def test_gray_rule_equals_cv2():
    img = np.random.default_rng(0).integers(0, 256, (97, 131, 3), dtype=np.uint8)
    assert np.array_equal(OG.gray(img), cv2.cvtColor(img, cv2.COLOR_RGB2GRAY))


def write_raw_set(root, seed=0):
    """Raw images as a user would have them: 640x480, 427x640 and 500x375 baseline JPEGs, a gray JPEG, a progressive
    JPEG, a PNG and a truncated file (skipped).  -> [readable flag per sorted name]."""
    rng = np.random.default_rng(seed)
    os.makedirs(root, exist_ok=True)

    def img(h, w):
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
        base = np.stack([128 + 80 * np.sin(xx / (7 + 5 * c)) * np.cos(yy / 9.0) for c in range(3)], -1)
        return np.clip(base + rng.normal(0, 12, base.shape), 0, 255).astype(np.uint8)

    files = {"a_640x480.jpg": (img(480, 640), []), "b_427x640.jpg": (img(640, 427), []), "c_500x375.jpg": (img(375, 500), []),
             "d_gray.jpg": (cv2.cvtColor(img(300, 400), cv2.COLOR_BGR2GRAY), []),
             "e_progressive.jpg": (img(480, 640), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]), "f_image.png": (img(200, 260), []),
             "h_640x480.jpg": (img(480, 640), [cv2.IMWRITE_JPEG_QUALITY, 80])}
    for name, (im, params) in files.items():
        cv2.imwrite(os.path.join(root, name), im, params)
    blob = open(os.path.join(root, "a_640x480.jpg"), "rb").read()
    with open(os.path.join(root, "g_truncated.jpg"), "wb") as f:
        f.write(blob[:300])                                            # cv2.imread returns None
    with open(os.path.join(root, ".hidden.jpg"), "wb") as f:
        f.write(blob)
    return [cv2.imread(os.path.join(root, n)) is not None for n in sorted(os.listdir(root)) if not n.startswith(".")]


def gen_args(tmp, mode, color=True, num_data=9, test_num_data=5, img_per_real=2, extra=()):
    from unsuperviseddeephomographyral2018_b200 import gen_data as G
    argv = ["--mode", mode, "--color", "true" if color else "false", "--raw_data_path", str(tmp / "raw"),
            "--test_raw_data_path", str(tmp / "raw"), "--data_path", str(tmp / "data") + "/", "--num_data", str(num_data),
            "--test_num_data", str(test_num_data), "--img_per_real", str(img_per_real)] + list(extra)
    return G.resolve_args(G.build_parser().parse_args(argv))


def _rows(path):
    with open(path) as f:
        return f.read()


@pytest.mark.parametrize("mode,num_data,img_per_real", [("train", 9, 2), ("train", 4, 3), ("test", 9, 2)])
def test_host_generator_draws_files_and_cutoffs_follow_the_reference(tmp_path, mode, num_data, img_per_real):
    from unsuperviseddeephomographyral2018_b200 import dataloader, gen_data as G
    readable = write_raw_set(tmp_path / "raw")
    assert readable.count(False) == 1
    args = gen_args(tmp_path, mode, num_data=num_data, img_per_real=img_per_real)
    end = G.generate(args, OG.HostBackend(), seed=5)
    start = num_data if mode == "test" else 0
    n = 5 if mode == "test" else num_data
    want = OG.reference_draws(readable, n, start, img_per_real, seed=5)
    assert end == start + len(want) and len(want) == min(n, readable.count(True) * img_per_real)
    pre = "test_" if mode == "test" else ""
    d = str(tmp_path / "data")
    gt = "".join("%s\n" % " ".join("%.18e" % v for v in np.subtract(np.array(p), np.array(f)).flatten().astype(np.float32))
                 for _, f, p in want)
    pts1 = "".join("%s\n" % " ".join("%.18e" % v for v in np.array(f).flatten().astype(np.float32)) for _, f, p in want)
    names = "".join("%d.jpg %d.jpg\n" % (i, i) for i, _, _ in want)
    assert _rows(os.path.join(d, pre + "gt.txt")) == gt
    assert _rows(os.path.join(d, pre + "pts1.txt")) == pts1
    assert _rows(os.path.join(d, pre + "synthetic.txt" if mode == "test" else "train_synthetic.txt")) == names
    assert sorted(os.listdir(os.path.join(d, "I"))) == sorted("%d.jpg" % i for i, _, _ in want)
    lst, p1, g1 = dataloader.read_img_and_gt(os.path.join(d, pre + "synthetic.txt" if mode == "test" else "train_synthetic.txt"),
                                             os.path.join(d, pre + "pts1.txt"), os.path.join(d, pre + "gt.txt"))
    assert len(lst) == len(want) and np.array_equal(np.asarray(p1, np.float64).reshape(-1, 8),
                                                    np.array([np.array(f).flatten() for _, f, _ in want], np.float64))


def test_resume_n_deletes_and_resume_y_appends(tmp_path):
    from unsuperviseddeephomographyral2018_b200 import gen_data as G
    write_raw_set(tmp_path / "raw")
    G.generate(gen_args(tmp_path, "train", num_data=4), OG.HostBackend(), seed=1)
    G.generate(gen_args(tmp_path, "train", num_data=3, extra=["--resume", "Y", "--start_index", "4"]), OG.HostBackend(), seed=2)
    d = str(tmp_path / "data")
    assert sorted(os.listdir(os.path.join(d, "I"))) == ["%d.jpg" % i for i in range(7)]
    assert len(_rows(os.path.join(d, "gt.txt")).splitlines()) == 7
    G.generate(gen_args(tmp_path, "train", num_data=2), OG.HostBackend(), seed=3)        # --resume N: start over
    assert sorted(os.listdir(os.path.join(d, "I"))) == ["0.jpg", "1.jpg"]
    assert len(_rows(os.path.join(d, "train_synthetic.txt")).splitlines()) == 2


def test_gray_files_only_in_train_mode_without_color(tmp_path):
    from unsuperviseddeephomographyral2018_b200 import gen_data as G
    write_raw_set(tmp_path / "raw")
    G.generate(gen_args(tmp_path, "train", color=False, num_data=2), OG.HostBackend(), seed=0)
    im = cv2.imread(str(tmp_path / "data" / "I" / "0.jpg"), cv2.IMREAD_UNCHANGED)
    assert im.ndim == 2
    G.generate(gen_args(tmp_path, "test", color=False, num_data=2, test_num_data=2), OG.HostBackend(), seed=0)
    assert cv2.imread(str(tmp_path / "data" / "I" / "2.jpg"), cv2.IMREAD_UNCHANGED).ndim == 3


def test_gen_warp_entry_rejects_bad_arguments():
    import ctypes
    from unsuperviseddeephomographyral2018_b200 import _lib
    L = _lib.lib
    p = ctypes.c_void_p(256)
    for i in (0, 1, 5, 6, 7):
        a = [p, p, 2, 240, 320, p, p, p, None]
        a[i] = None
        assert L.udh_gen_warp_u8(*a) == _lib.EINVAL
        assert b"null pointer" in L.udh_last_error()
    for n, h, w in ((-1, 240, 320), (70000, 240, 320), (2, 0, 320), (2, 240, 0)):
        assert L.udh_gen_warp_u8(p, p, n, h, w, p, p, p, None) == _lib.EINVAL
        assert b"bad dimensions" in L.udh_last_error()
