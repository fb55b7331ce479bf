"""CPU tests of the alignment API's host logic: the coordinate convention against the real-data test metric, the pair list,
and align_images.py's defaults and homographies.txt format with a stub estimator."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_image_homography_is_the_real_metric_rule():
    """H x1 equals correspondence_errors' pred_corr2 when both images are r times the network size."""
    from unsuperviseddeephomographyral2018_b200 import align, real_metrics as rm
    rng = np.random.default_rng(11)
    for img_h, img_w in ((142, 190), (240, 320)):
        for r in (1.0, 1.5, 2.0, 2.5):                         # aspect-preserving: the metric scales both axes by one r
            B = 40
            x0, y0 = rng.integers(4, img_w - 132, B), rng.integers(4, img_h - 132, B)
            pts1 = np.stack([x0, y0, x0 + 128, y0, x0 + 128, y0 + 128, x0, y0 + 128], 1).astype(np.float32)
            h4p = rng.normal(0, 8, (B, 8)).astype(np.float32)
            size = (int(img_h * r), int(img_w * r))
            c1 = rng.uniform(10, min(size) - 10, (B, 8))
            gt = np.concatenate([c1, c1 + rng.normal(0, 5, (B, 8))], 1)
            errs = rm.correspondence_errors(h4p, pts1, gt, full_img_h=size[0], img_h=img_h, corr_scale=1.0, with_points=True)
            H = align.image_homography(h4p, pts1, size, size, img_h, img_w)
            assert H.dtype == np.float64 and np.allclose(H[:, 2, 2], 1.0, rtol=0, atol=0)
            for k in range(B):
                got = rm.perspective_transform(c1[k].reshape(4, 2), H[k])
                ref = errs[k][3]
                assert np.all(np.abs(got - ref) <= 1e-9 * np.abs(ref)), (img_h, r, k, got, ref)


def test_image_homography_maps_the_patch_corners_with_separate_scales():
    """Different image sizes: H takes image 1's corners S_1 (pts1 + h4p) to image 2's S_2 pts1."""
    from unsuperviseddeephomographyral2018_b200 import align, real_metrics as rm
    rng = np.random.default_rng(3)
    pts1 = np.array([[31, 7, 159, 7, 159, 135, 31, 135]], np.float32)
    h4p = rng.normal(0, 6, (1, 8)).astype(np.float32)
    s1, s2 = (3000, 4000), (480, 640)
    H = align.image_homography(h4p, pts1, s1, s2, 142, 190)[0]
    c1 = (pts1 + h4p).reshape(4, 2).astype(np.float64) * [4000 / 190.0, 3000 / 142.0]
    c2 = pts1.reshape(4, 2).astype(np.float64) * [640 / 190.0, 480 / 142.0]
    assert np.allclose(rm.perspective_transform(c1, H), c2, rtol=0, atol=1e-3)


def test_centred_corners():
    from unsuperviseddeephomographyral2018_b200 import align
    assert align.centred_corners(2, 142, 190, 128).tolist() == [[31, 7, 159, 7, 159, 135, 31, 135]] * 2
    assert align.centred_corners(1, 240, 320, 128)[0].tolist() == [96, 56, 224, 56, 224, 184, 96, 184]


def test_prep_path_follows_the_area_rule():
    from unsuperviseddeephomographyral2018_b200 import align
    assert align.prep_path(240, 320, 240, 320) == align.PREP_DEVICE
    assert align.prep_path(1080, 1920, 240, 320) == align.PREP_DEVICE
    assert align.prep_path(3000, 4000, 240, 320) == align.PREP_DEVICE          # source rows read from global memory
    assert align.prep_path(3000, 4000, 142, 190) == align.PREP_DEVICE
    assert align.prep_path(480, 640, 240, 320) == align.PREP_HOST              # integer ratio: resizeAreaFast
    assert align.prep_path(100, 150, 142, 190) == align.PREP_DEVICE_UPSCALE
    assert align.prep_path(100, 400, 142, 190) == align.PREP_HOST


def test_read_pairs_resolves_paths_against_the_list(tmp_path):
    from unsuperviseddeephomographyral2018_b200 import align
    (tmp_path / "sub").mkdir()
    lst = tmp_path / "sub" / "pairs.txt"
    lst.write_text("a.jpg b.jpg\n\n x/c.png  d.png \n")
    names, paths = align.read_pairs(str(lst))
    assert names == [("a.jpg", "b.jpg"), ("x/c.png", "d.png")]
    assert paths[1] == (str(tmp_path / "sub" / "x" / "c.png"), str(tmp_path / "sub" / "d.png"))
    lst.write_text("a.jpg\n")
    with pytest.raises(ValueError):
        align.read_pairs(str(lst))


def test_cli_defaults():
    import align_images as cli
    import homography_CNN_synthetic as syn
    a = cli.build_parser().parse_args(["--img1", "a.jpg", "--img2", "b.jpg"])
    assert (a.img_h, a.img_w, a.patch_size, a.numeric, a.batch_size, a.save_warped, a.seed, a.model_name, a.loss_type,
            a.seeded_weights) == (240, 320, 128, "bf16x3", 128, True, 0, "model.ckpt", "l1_loss", False)
    # the same --model_dir / --loss_type name the same directory as homography_CNN_synthetic.py --mode test
    for argv in ([], ["--model_dir", "/x/models", "--loss_type", "h_loss"]):
        s = syn.resolve_paths(syn.build_parser().parse_args(["--mode", "test"] + argv))
        assert cli.checkpoint_dir(cli.build_parser().parse_args(argv)) == s.model_dir
    assert cli.build_parser().parse_args(["--pairs", "p", "--save_warped", "False"]).save_warped is False


class StubEstimator(object):
    """estimate() returns a fixed homography per pair built from the pair's index; no device."""

    def __init__(self):
        self.calls = []
        self.last_ms = {}

    def estimate(self, I1, I2):
        self.calls.append(len(I1))
        H = np.stack([np.array([[1.0, 1e-3 * k, 10.0 / 3], [0, 2.0 ** -20, -1234.56789], [1e-7, -2e-6, 1.0]]) for k in range(len(I1))])
        self.last_ms = dict(prep=1.0, forward=2.0)
        return H, None, None


def test_cli_writes_homographies_txt(tmp_path, capsys):
    import align_images as cli
    lst = tmp_path / "pairs.txt"
    lst.write_text("".join("i%d.jpg p%d.jpg\n" % (k, k) for k in range(5)))
    args = cli.build_parser().parse_args(["--pairs", str(lst), "--out_dir", str(tmp_path / "out"), "--save_warped", "False",
                                          "--batch_size", "2"])
    est = StubEstimator()
    decoded = []
    decode = lambda paths: decoded.append(paths) or [np.zeros((4, 6, 3), np.uint8) for _ in paths]
    written = cli.run(args, est, decode, None)
    assert est.calls == [2, 2, 1]
    assert decoded[0] == [str(tmp_path / "i0.jpg"), str(tmp_path / "p0.jpg"), str(tmp_path / "i1.jpg"), str(tmp_path / "p1.jpg")]
    lines = (tmp_path / "out" / "homographies.txt").read_text().splitlines()
    assert len(lines) == 5
    for k, ln in enumerate(lines):
        parts = ln.split(" ")
        assert parts[:2] == ["i%d.jpg" % k, "p%d.jpg" % k] and len(parts) == 11
        vals = np.array([float(v) for v in parts[2:]]).astype(np.float32)
        H = np.array([[1.0, 1e-3 * (k % 2), 10.0 / 3], [0, 2.0 ** -20, -1234.56789], [1e-7, -2e-6, 1.0]])
        assert np.array_equal(vals, H.reshape(-1).astype(np.float32))          # '%.9g' reads back to the float32 values
        assert np.array_equal(written[k], vals)
        assert parts[2:] == ["%.9g" % v for v in H.reshape(-1).astype(np.float32)]
    assert "GPU" in capsys.readouterr().out


def test_cli_stops_without_a_checkpoint(tmp_path):
    import align_images as cli
    args = cli.build_parser().parse_args(["--img1", "a", "--img2", "b", "--model_dir", str(tmp_path)])
    with pytest.raises(SystemExit) as e:
        cli.make_estimator(args)
    assert "no checkpoint" in str(e.value) and "--seeded_weights" in str(e.value)


def test_check_corners_accepts_only_integer_squares_inside_the_frame():
    from unsuperviseddeephomographyral2018_b200 import align
    good = align.centred_corners(3, 142, 190, 128)
    good[1] = [0, 0, 128, 0, 128, 128, 0, 128]
    good[2] = [62, 14, 190, 14, 190, 142, 62, 142]                      # touching the right and bottom edges
    assert np.array_equal(align.check_corners(good, 3, 142, 190, 128), good)
    for bad in ([-1, 7, 127, 7, 127, 135, -1, 135],                     # left of the frame
                [63, 7, 191, 7, 191, 135, 63, 135],                     # right of the frame
                [31, 15, 159, 15, 159, 143, 31, 143],                   # below the frame
                [31.5, 7, 159.5, 7, 159.5, 135, 31.5, 135],             # not integer
                [31, 7, 159, 7, 160, 135, 31, 135],                     # not a square
                [31, 7, 159, 7, 159, 135, 31, float("nan")]):
        c = good.copy(); c[1] = bad
        with pytest.raises(ValueError):
            align.check_corners(c, 3, 142, 190, 128)
    with pytest.raises(ValueError):
        align.check_corners(good[:2], 3, 142, 190, 128)                 # wrong count
