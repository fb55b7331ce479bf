"""GPU tests of the report image (--save_visual): the device canvas against oracle/draw.py and cv2 on the seeded vertex
sets of tests/test_draw_oracle.py, the denormalised images (with and without augmentation) against a host restatement,
the JPEG bytes against cv2.imencode, and the files of the three test harnesses end to end.

Deliberate faults, injected one at a time, and the tests that failed (one H100, 400 W):
  prediction polygon drawn after stacking (not clipped to img2)   test_canvas_equals_oracle_and_cv2: 13 of 16 cases
  a match's LINE_AA line drawn after its first circle              test_canvas_equals_oracle_and_cv2 (16 of 16),
                                                                  test_jpeg_bytes_equal_cv2_imencode,
                                                                  test_report_files_of_the_synthetic_cli[True]
  circle polygon one vertex short (12 of 13)                       the same three
  end2 rounded half-up (report.py, CPU)                            test_report_logic::test_conversions,
                                                                  test_draw_oracle::test_composition (4 of 4)
  kp1 rounded instead of truncated (report.py, CPU)                the same two"""
import glob
import os
import pathlib
import subprocess
import sys

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from oracle import draw as D  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _aug_table(rng, B):
    """[B,11] augmentation rows as udh_prep_inputs_u8_ex reads them: flag, then (gamma, brightness, 3 gains) per image."""
    a = np.zeros((B, 11), np.float32)
    a[:, 0] = 1.0
    for im in range(2):
        a[:, 1 + 5 * im] = rng.uniform(0.8, 1.2, B)
        a[:, 2 + 5 * im] = rng.uniform(0.5, 2.0, B)
        a[:, 3 + 5 * im:6 + 5 * im] = rng.uniform(0.8, 1.2, (B, 3))
    return a


@pytest.mark.parametrize("B", [1, 7, 128, 129])
@pytest.mark.parametrize("use_aug", [False, True], ids=["noaug", "aug"])
@pytest.mark.parametrize("prime_left", [True, False], ids=["Iprime_left", "I_left"])
def test_canvas_equals_oracle_and_cv2(B, use_aug, prime_left):
    from unsuperviseddeephomographyral2018_b200 import ops
    h, w = (17, 23) if B != 128 else (48, 64)
    rng = np.random.default_rng(1000 * B + 10 * use_aug + prime_left)
    I = rng.integers(0, 256, (B, h, w, 3), np.uint8)
    Ip = rng.integers(0, 256, (B, h, w, 3), np.uint8)
    Ip[::3] = 90                                                   # constant backgrounds too
    verts = D.vertex_cases(rng, B, h, w)
    aug = _aug_table(rng, B) if use_aug else None
    aug_t = torch.from_numpy(aug).cuda() if use_aug else None
    got = ops.draw_report_u8(torch.from_numpy(I).cuda(), torch.from_numpy(Ip).cuda(), aug_t, torch.from_numpy(verts).cuda(), prime_left)
    got = got.cpu().numpy()
    # the denormalised images the kernel starts from, against the host restatement (each image with its own aug row)
    zero = np.full((B, 20, 2), -(1 << 31), np.int32)                # every primitive far outside: the bare canvas
    base = ops.draw_report_u8(torch.from_numpy(I).cuda(), torch.from_numpy(Ip).cuda(), aug_t, torch.from_numpy(zero).cuda(), prime_left).cpu().numpy()
    for k in range(B):
        row = aug[k] if use_aug else None
        dI, dIp = D.host_denorm(I[k], row, 0), D.host_denorm(Ip[k], row, 1)
        left, right = (dIp, dI) if prime_left else (dI, dIp)
        np.testing.assert_array_equal(base[k, :, :w], left, err_msg="sample %d left image" % k)
        np.testing.assert_array_equal(base[k, :, w:], right, err_msg="sample %d right image" % k)
    for k in range(B):
        img1, img2 = base[k, :, :w], base[k, :, w:]
        ref = D.cv2_draw_report(img1, img2, verts[k])
        assert np.array_equal(got[k], ref), "sample %d verts %s: %d pixels differ from cv2" % (k, verts[k].tolist(), int((got[k] != ref).any(-1).sum()))
        if k < 24:
            assert np.array_equal(D.draw_report(img1, img2, verts[k]), ref)


def test_jpeg_bytes_equal_cv2_imencode():
    from unsuperviseddeephomographyral2018_b200 import ops
    B, h, w = 16, 240, 320
    rng = np.random.default_rng(77)
    I = rng.integers(0, 256, (B, h, w, 3), np.uint8)
    Ip = rng.integers(0, 256, (B, h, w, 3), np.uint8)
    c1 = rng.uniform(20, 300, (B, 4, 2)).astype(np.float32)
    c2 = (c1 + rng.normal(0, 10, (B, 4, 2))).astype(np.float32)
    pr = (c2 + rng.normal(0, 5, (B, 4, 2))).astype(np.float32)
    from unsuperviseddeephomographyral2018_b200 import report
    verts = np.stack([report.report_vertices(a, b, c, w) for a, b, c in zip(c1, c2, pr)])
    canv = ops.draw_report_u8(torch.from_numpy(I).cuda(), torch.from_numpy(Ip).cuda(), None, torch.from_numpy(verts).cuda(), True)
    blobs = ops.encode_jpeg(canv, quality=95)
    for k in range(B):
        ref = D.cv2_draw_report(D.host_denorm(Ip[k]), D.host_denorm(I[k]), verts[k])
        assert blobs[k] == cv2.imencode(".jpg", ref)[1].tobytes(), k


@pytest.mark.parametrize("save_visual", ["True", "False"])
def test_report_files_of_the_synthetic_cli(tmp_path, save_visual):
    """`--mode test --synthetic 16 --batch_size 4`: 12 files named as the reference names them, each the cv2 composition of
    the same seeded batch with the engine's own prediction; --save_visual False writes none."""
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl, engine as en, report
    seed, nb, bs = 3, 16, 4
    res = tmp_path / "r"
    cmd = [sys.executable, os.path.join(ROOT, "homography_CNN_synthetic.py"), "--mode", "test", "--batch_size", str(bs), "--synthetic", str(nb),
           "--num_gpus", "1", "--numeric", "bf16x3", "--seed", str(seed), "--do_augment", "0", "--model_dir", str(tmp_path / "m"),
           "--log_dir", str(tmp_path / "l"), "--results_dir", str(res), "--save_visual", save_visual]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    files = sorted(os.listdir(res)) if res.exists() else []
    if save_visual == "False":
        assert files == []
        return
    assert len(files) == 3 * (nb // bs) and r.stdout.count("Wrote file %s") == len(files)
    dparams = dl.dataloader_params(data_path="", filenames_file=None, pts1_file=None, gt_file=None, mode='test', batch_size=bs, img_h=240,
                                   img_w=320, patch_size=128, augment_list=['normalize'], do_augment=0.0)
    loader = dl.Dataloader(dparams, shuffle=True, synthetic_pairs=nb, seed=seed * 97 + 12345, device="cuda")
    eng = en.HomographyEngine(bs, 128, 240, 320, numeric="bf16x3", seed=seed, loss_type="l1_loss")
    seen = set()
    for step in range(3 * (nb // bs)):
        b = loader.next_batch()
        out = eng.eval_step(b)
        h = eng.losses_dict(out)["bounded_h_loss"]
        name = report.synthetic_name(step, bs, "l1_loss", h)
        assert name.startswith("%d_l1_loss_loss_" % (step * bs)) and name in files, (name, files)
        seen.add(name)
        c1, c2, pr = report.synthetic_points(b["pts1"][:1].cpu().numpy(), b["gt"][:1].cpu().numpy(), out["pred_h4p"][:1].cpu().numpy())
        img1, img2 = D.host_denorm(b["I_prime_u8"][0].cpu().numpy()), D.host_denorm(b["I_u8"][0].cpu().numpy())
        kp2 = (c2[0] + np.array([320, 0])).astype(np.int32)
        kp1 = c1[0].astype(np.int32)
        end2 = np.round(c2[0]).astype(int) + np.array([320, 0])
        with np.errstate(invalid="ignore"):
            v = np.concatenate([np.int32(pr[0]), kp2, kp1, kp1, end2]).astype(np.int32)
        ref = D.cv2_draw_report(img1, img2, v)
        assert (res / name).read_bytes() == cv2.imencode(".jpg", ref)[1].tobytes(), name
    assert seen == set(files)


def _jpgs(d):
    return sorted(os.path.basename(f) for f in glob.glob(os.path.join(str(d), "*.jpg")))


def _check_files(res, b, i, name, corr1, corr2, pred, prime_left):
    aug = b["aug"].cpu().numpy()[i] if b.get("aug") is not None else None
    dI, dIp = D.host_denorm(b["I_u8"][i].cpu().numpy(), aug, 0), D.host_denorm(b["I_prime_u8"][i].cpu().numpy(), aug, 1)
    img1, img2 = (dIp, dI) if prime_left else (dI, dIp)
    with np.errstate(invalid="ignore"):
        ref = D.cv2_compose(img1, img2, corr1, corr2, pred)
    assert (res / name).read_bytes() == cv2.imencode(".jpg", ref)[1].tobytes(), name


@pytest.mark.parametrize("save_visual", ["True", "False"])
def test_report_files_of_the_real_cnn_cli(tmp_path, save_visual):
    """`homography_CNN_real.py --mode test --synthetic 16 --batch_size 8` (augmentation on): one file per sample, named
    <k>_Unsupervised__loss_<h_loss>.jpg, each the cv2 composition of the full-size images with the clicked points and the
    predicted matches that the metric computes."""
    import importlib
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl, engine as en, real_metrics as rm, report
    sys.path.insert(0, ROOT)
    R = importlib.import_module("homography_CNN_real")
    argv = ["--mode", "test", "--synthetic", "16", "--batch_size", "8", "--num_gpus", "1", "--seed", "4", "--numeric", "bf16x3",
            "--load_model_dir", str(tmp_path / "m") + "/", "--save_model_dir", str(tmp_path / "s") + "/", "--log_dir", str(tmp_path / "l") + "/",
            "--results_dir", str(tmp_path / "r") + "/", "--save_visual", save_visual]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "homography_CNN_real.py")] + argv, capture_output=True, text=True, timeout=900,
                       cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    args = R.resolve_paths(R.build_parser().parse_args(argv))
    res = pathlib.Path(args.results_dir)
    files = _jpgs(res)
    if save_visual == "False":
        assert files == []
        return
    assert len(files) == 16 and r.stdout.count("Wrote file %s") == 16
    loader = dl.Dataloader(R.loader_params(args, 'test', 8), shuffle=False, synthetic_pairs=16, seed=4 * 97 + 12345, device="cuda", rho=R.RHO)
    eng = en.HomographyEngine(8, args.patch_size, args.img_h, args.img_w, numeric="bf16x3", seed=4, loss_type=args.loss_type)
    names = []
    for step in range(2):
        b = loader.next_batch()
        out = eng.eval_step(b)
        errs = rm.correspondence_errors(out["pred_h4p"].cpu().numpy(), b["pts1"].cpu().numpy(), b["gt_corr"], full_img_h=args.full_img_h,
                                        img_h=args.img_h, with_points=True)
        corr1, corr2 = report.clicked_points(b["gt_corr"])
        for i, e in enumerate(errs):
            name = "%d_Unsupervised__loss_%s.jpg" % (step * 8 + i, str(e[0]))
            names.append(name)
            _check_files(res, b, i, name, corr1[i], corr2[i], e[3], prime_left=False)
    assert sorted(names) == files


@pytest.mark.parametrize("method", ["direct", "identity"])
def test_report_files_of_the_conventional_real_cli(tmp_path, method):
    """`homography_conventional_real.py --method direct|identity --synthetic 16 --batch_size 8` (augmentation on): one file
    per pair, named <k>_loss_<h_loss>.jpg, each the cv2 composition with pred_h4p (clamped to +-80) + corr1."""
    import importlib
    from unsuperviseddeephomographyral2018_b200 import report
    sys.path.insert(0, ROOT)
    M = importlib.import_module("homography_conventional_real")
    argv = ["--method", method, "--synthetic", "16", "--batch_size", "8", "--num_iterations", "20", "--do_augment", "0.5",
            "--log_dir", str(tmp_path / "l"), "--results_dir", str(tmp_path / "r")]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "homography_conventional_real.py")] + argv, capture_output=True, text=True,
                       timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    args = M.resolve_paths(M.build_parser().parse_args(argv))
    res = pathlib.Path(args.results_dir)
    files = _jpgs(res)
    assert len(files) == 16 and r.stdout.count("Wrote file %s") == 16
    loader = M.make_loader(args, 8)
    names = []
    for step in range(2):
        b = loader.next_batch()
        h, f, _, pred = M.run_batch(method, b, 20)
        corr1, corr2 = report.clicked_points(b["gt_corr"])
        for i in range(8):
            name = "%d_loss_%s.jpg" % (step * 8 + i, str(float(h[i])))
            names.append(name)
            _check_files(res, b, i, name, corr1[i], corr2[i], pred[i].reshape(4, 2) + corr1[i], prime_left=False)
    assert sorted(names) == files


def test_conventional_real_save_visual_false_writes_no_image(tmp_path):
    argv = ["--method", "identity", "--synthetic", "8", "--batch_size", "8", "--log_dir", str(tmp_path / "l"), "--results_dir",
            str(tmp_path / "r"), "--save_visual", "False"]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "homography_conventional_real.py")] + argv, capture_output=True, text=True,
                       timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert glob.glob(str(tmp_path / "r" / "**" / "*.jpg"), recursive=True) == [] and "Wrote file" not in r.stdout
