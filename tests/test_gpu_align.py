"""GPU tests of image alignment: udh_warp_perspective_u8 against cv2 and its restatement, the estimator's batch against the
real-data loader's, batch invariance, the geometry against the real-data test metric, mixed sizes, and align_images.py end
to end."""
import os
import sys

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import jpeg as J  # noqa: E402
from oracle import warp_perspective as WP  # noqa: E402
from test_warp_perspective_oracle import SIZES, named_matrices  # noqa: E402

pytestmark = pytest.mark.gpu


def _bits(t):
    return np.asarray(t.cpu() if isinstance(t, torch.Tensor) else t, np.float32).view(np.uint32)


# ---- the warp kernel -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("channels", [1, 3], ids=["gray", "bgr"])
@pytest.mark.parametrize("src_hw,dst_hw", SIZES, ids=["%dx%d_to_%dx%d" % (a + b) for a, b in SIZES])
def test_warp_kernel_equals_cv2(channels, src_hw, dst_hw):
    from unsuperviseddeephomographyral2018_b200 import ops
    (h, w), (dh, dw) = src_hw, dst_hw
    rng = np.random.default_rng(h * 1000 + w + dh + channels)
    mats = named_matrices(h, w, dh, dw)
    src = rng.integers(0, 256, (len(mats), h, w, channels), np.uint8)
    M = np.stack(list(mats.values()))
    got = ops.warp_perspective_u8(torch.from_numpy(src).cuda(), torch.from_numpy(M).cuda(), dh, dw).cpu().numpy()
    for k, name in enumerate(mats):
        ref = cv2.warpPerspective(src[k] if channels == 3 else src[k, ..., 0], M[k], (dw, dh)).reshape(dh, dw, channels)
        assert np.array_equal(got[k], ref), name


def test_warp_kernel_camera_frame_and_mixed_batch():
    from unsuperviseddeephomographyral2018_b200 import ops
    rng = np.random.default_rng(12)
    frame = J.textured(rng, 3000, 4000, 3)
    M = np.array([[0.98, 0.05, 40.0], [-0.04, 1.01, -25.0], [2e-6, -1e-5, 1.0]])
    got = ops.warp_perspective_u8(torch.from_numpy(frame[None]).cuda(), torch.from_numpy(M[None]).cuda(), 3000, 4000)
    assert np.array_equal(got[0].cpu().numpy(), cv2.warpPerspective(frame, M, (4000, 3000)))
    B, h, w = 24, 120, 170
    src = rng.integers(0, 256, (B, h, w, 3), np.uint8)
    Ms = np.eye(3) + rng.normal(0, 0.1, (B, 3, 3)) * [[1, 1, 20], [1, 1, 20], [0.003, 0.003, 0.1]]
    Ms[3] = [[1, 0, 0], [0, 1, 0], [0.125, 0, 1.0]]
    Ms[7] = [[1, 2, 0], [2, 4, 0], [0, 0, 1.0]]
    got = ops.warp_perspective_u8(torch.from_numpy(src).cuda(), torch.from_numpy(Ms).cuda(), 97, 211).cpu().numpy()
    for k in range(B):
        assert np.array_equal(got[k], cv2.warpPerspective(src[k], Ms[k], (211, 97))), k
        assert np.array_equal(got[k], WP.warp_perspective(src[k], Ms[k], (211, 97))), k


def test_warp_rejects_bad_arguments():
    from unsuperviseddeephomographyral2018_b200 import _lib, ops
    src = torch.zeros(2, 8, 8, 3, dtype=torch.uint8, device="cuda")
    with pytest.raises(_lib.UdhError):
        ops.warp_perspective_u8(src, torch.zeros(1, 3, 3, dtype=torch.float64, device="cuda"), 8, 8)
    with pytest.raises(_lib.UdhError):
        ops.warp_perspective_u8(torch.zeros(2, 8, 8, 2, dtype=torch.uint8, device="cuda"), torch.zeros(2, 3, 3, dtype=torch.float64, device="cuda"), 8, 8)
    with pytest.raises(_lib.UdhError):
        ops.warp_perspective_u8(src, torch.zeros(2, 3, 3, dtype=torch.float32, device="cuda"), 8, 8)


# ---- the estimator against the real-data loader -------------------------------------------------------------------------------
def _write_set(root, sizes, n, net=(142, 190), P=128, corners="centred", seed=0, gt=False):
    """I/, I_prime/ JPEG pairs (sizes cycled), test_real.txt, test_pts1.txt (centred patch, or seeded ones), and with gt four
    clicked correspondences per pair on frames twice the file size."""
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "I")); os.makedirs(os.path.join(root, "I_prime"))
    names, pts1, corr = [], [], []
    for i in range(n):
        hh, ww = sizes[i % len(sizes)]
        name = "%06d.jpg" % (i + 1)
        base = J.textured(rng, hh, ww, 3)
        M = np.array([[1, 0.02, 3.0], [-0.01, 1, -2.0], [1e-5, 0, 1.0]])
        for sub, img in (("I", base), ("I_prime", cv2.warpPerspective(base, M, (ww, hh), borderMode=cv2.BORDER_REFLECT))):
            cv2.imwrite(os.path.join(root, sub, name), img[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, 95])
        names.append("%s %s" % (name, name))
        if corners == "centred":
            x0, y0 = (net[1] - P) // 2, (net[0] - P) // 2
        else:
            x0, y0 = rng.integers(4, net[1] - P - 3), rng.integers(4, net[0] - P - 3)
        pts1.append([x0, y0, x0 + P, y0, x0 + P, y0 + P, x0, y0 + P])
        c1 = rng.uniform(40, 2 * min(hh, ww) - 40, 8)
        corr.append(np.concatenate([c1, c1 + rng.normal(0, 6, 8)]))
    with open(os.path.join(root, "test_real.txt"), "w") as f:
        f.write("\n".join(names) + "\n")
    np.savetxt(os.path.join(root, "test_pts1.txt"), np.array(pts1, np.float64))
    if gt:
        np.savetxt(os.path.join(root, "test_gt.txt"), np.array(corr, np.float64))
    return [(os.path.join(root, "I", nm.split()[0]), os.path.join(root, "I_prime", nm.split()[0])) for nm in names]


def _loader(root, B, net, full, gt=False):
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl
    prm = dl.extended_dataloader_params(data_path=str(root), filenames_file=os.path.join(root, "test_real.txt"),
                                        pts1_file=os.path.join(root, "test_pts1.txt"),
                                        gt_file=os.path.join(root, "test_gt.txt") if gt else None, mode="test", batch_size=B,
                                        img_h=net[0], img_w=net[1], patch_size=128, augment_list=["normalize"], do_augment=0.0,
                                        full_img_h=full[0], full_img_w=full[1])
    return dl.Dataloader(prm, shuffle=False, seed=3, device="cuda")


@pytest.mark.parametrize("numeric", ["fp32", "bf16", "bf16x3"])
def test_estimate_batch_equals_the_loader(tmp_path, numeric):
    from unsuperviseddeephomographyral2018_b200 import align, engine
    net, full, B = (142, 190), (240, 320), 8
    paths = _write_set(tmp_path, [full], B)
    b = _loader(tmp_path, B, net, full).next_batch()
    imgs = align.decode_images([p for pr in paths for p in pr])
    I1, I2 = torch.stack(imgs[0::2]), torch.stack(imgs[1::2])
    assert torch.equal(I1, b["I_u8"]) and torch.equal(I2, b["I_prime_u8"])
    eng = engine.HomographyEngine(B, 128, net[0], net[1], numeric=numeric, seed=5)
    est = align.HomographyEstimator(engine=eng)
    mine = est.prepare(I1, I2)
    assert est.prep_paths == {full: align.PREP_DEVICE}
    for k in ("I1_aug", "I2_aug", "I_aug", "I_prime_aug", "I1", "I2", "pts1"):
        assert np.array_equal(_bits(mine[k]), _bits(b[k])), k
    assert torch.equal(mine["patch_indices"], b["patch_indices"])
    ref = eng.forward(b, train=False)["pred_h4p"].cpu().numpy()
    H, h4p, pts1 = est.estimate(I1, I2)
    assert np.array_equal(_bits(h4p), _bits(ref))
    assert np.array_equal(pts1, b["pts1"].cpu().numpy())
    assert np.array_equal(H, align.image_homography(ref, pts1, full, full, net[0], net[1]))


def test_batch_invariance(tmp_path):
    from unsuperviseddeephomographyral2018_b200 import align
    rng = np.random.default_rng(4)
    est = align.HomographyEstimator(batch_size=128, seed=2)
    pool = [torch.from_numpy(J.textured(rng, 240, 320, 3)).cuda() for _ in range(40)]
    X1, X2 = pool[0], pool[1]
    H_alone = est.estimate([X1], [X2])[0][0]
    for pos in (0, 57, 127):
        L1 = [pool[(3 * k + 2) % 40] for k in range(128)]
        L2 = [pool[(5 * k + 7) % 40] for k in range(128)]
        L1[pos], L2[pos] = X1, X2
        assert np.array_equal(est.estimate(L1, L2)[0][pos], H_alone), pos
    L1 = [pool[k % 40] for k in range(131)]
    L2 = [pool[(k + 1) % 40] for k in range(131)]
    L1[129], L2[129] = X1, X2                                             # in the padded last batch of 3
    assert np.array_equal(est.estimate(L1, L2)[0][129], H_alone)


def test_geometry_matches_the_real_metric(tmp_path):
    """A real-mode engine (142 x 190) on a set whose files are twice the network size: H x1 of every pair equals the real
    test metric's pred_corr2 on the loader's batch."""
    from unsuperviseddeephomographyral2018_b200 import align, engine, real_metrics as rm
    net, full, B = (142, 190), (284, 380), 16
    paths = _write_set(tmp_path, [full], B, corners="seeded", gt=True)
    b = _loader(tmp_path, B, net, full, gt=True).next_batch()
    eng = engine.HomographyEngine(B, 128, net[0], net[1], numeric="bf16x3", seed=9)
    errs = rm.correspondence_errors(eng.forward(b, train=False)["pred_h4p"].cpu().numpy(), b["pts1"].cpu().numpy(), b["gt_corr"],
                                    full_img_h=full[0], img_h=net[0], with_points=True)
    est = align.HomographyEstimator(engine=eng)
    imgs = align.decode_images([p for pr in paths for p in pr])
    H, _, _ = est.estimate(imgs[0::2], imgs[1::2], corners=b["pts1"].cpu().numpy())
    assert est.prep_paths == {full: align.PREP_HOST}                       # integer ratio: the loader's host fallback
    for k in range(B):
        c1 = b["gt_corr"][k, :8].astype(np.float64).reshape(4, 2) * 0.5
        got = rm.perspective_transform(c1, H[k])
        assert np.abs(got - errs[k][3]).max() < 1e-4, k


def test_mixed_sizes_in_one_run():
    from unsuperviseddeephomographyral2018_b200 import align, dataloader as dl, ops
    rng = np.random.default_rng(8)
    sizes = [(240, 320), (480, 640), (1080, 1920), (3000, 4000)]
    est = align.HomographyEstimator(batch_size=4, seed=1)
    L1 = [torch.from_numpy(J.textured(rng, *sizes[k % 4], 3)).cuda() for k in range(8)]
    L2 = [torch.from_numpy(J.textured(rng, *sizes[(k + 1) % 4], 3)).cuda() for k in range(8)]
    H, h4p, _ = est.estimate(L1, L2)
    assert {s: est.prep_paths[s] for s in sizes} == {(240, 320): align.PREP_DEVICE, (480, 640): align.PREP_HOST,
                                                     (1080, 1920): align.PREP_DEVICE, (3000, 4000): align.PREP_DEVICE}
    for s in sizes:
        if ops.area_is_generic(s[0], s[1], 240, 320):
            # the device path's planes equal the loader's host arithmetic (cv2.resize INTER_AREA) for this size
            I = L1[sizes.index(s)][None]
            host = dl.normalise_resize_host(I[0].cpu().numpy().astype(np.float32), 240, 320)
            assert np.array_equal(_bits(est._planes(I)[0]), _bits(host)), s
    assert np.isfinite(H).all()
    for k in range(8):                                                    # each pair alone gives the same result
        assert np.array_equal(est.estimate([L1[k]], [L2[k]])[0][0], H[k]), k


# ---- the CLI ---------------------------------------------------------------------------------------------------------------------
def test_cli_end_to_end(tmp_path):
    import align_images as cli
    from unsuperviseddeephomographyral2018_b200 import align
    rng = np.random.default_rng(21)
    data = tmp_path / "data"
    (data / "a").mkdir(parents=True)
    lines = []
    for k, (s1, s2) in enumerate([((240, 320), (240, 320)), ((480, 640), (300, 400)), ((240, 320), (142, 190)), ((240, 320), (240, 320)),
                                  ((200, 260), (240, 320))]):
        n1, n2 = "a/%d_1.jpg" % k, "%d_2.%s" % (k, "png" if k == 3 else "jpg")
        cv2.imwrite(str(data / n1), J.textured(rng, *s1, 3), [cv2.IMWRITE_JPEG_QUALITY, 95])
        cv2.imwrite(str(data / n2), J.textured(rng, *s2, 3))
        lines.append("%s %s" % (n1, n2))
    (data / "pairs.txt").write_text("\n".join(lines) + "\n")
    outs = []
    for run in range(2):
        out = tmp_path / ("out%d" % run)
        assert cli.main(["--pairs", str(data / "pairs.txt"), "--out_dir", str(out), "--batch_size", "4", "--model_dir",
                         str(tmp_path / "no_model"), "--seeded_weights", "True", "--seed", "3"]) == 0
        outs.append(out)
    names = sorted(os.listdir(outs[0]))
    assert names == sorted(["homographies.txt"] + ["%d_warped.jpg" % k for k in range(5)])
    for nm in names:
        assert (outs[0] / nm).read_bytes() == (outs[1] / nm).read_bytes(), nm
    est = align.HomographyEstimator(batch_size=4, seed=3)
    paths = [str(data / p) for ln in lines for p in ln.split()]
    imgs = align.decode_images(paths)
    H, _, _ = est.estimate(imgs[0::2], imgs[1::2])
    txt = (outs[0] / "homographies.txt").read_text().splitlines()
    for k, ln in enumerate(txt):
        assert ln == align.format_line(*lines[k].split(), H[k])
        Hw = np.array([float(v) for v in ln.split()[2:]]).astype(np.float32).astype(np.float64).reshape(3, 3)
        img1, img2 = cv2.imread(paths[2 * k]), cv2.imread(paths[2 * k + 1])
        ok, ref = cv2.imencode(".jpg", cv2.warpPerspective(img1, Hw, (img2.shape[1], img2.shape[0])), [cv2.IMWRITE_JPEG_QUALITY, 95])
        assert (outs[0] / ("%d_warped.jpg" % k)).read_bytes() == ref.tobytes(), k


@pytest.mark.parametrize("net", [(240, 320), (142, 190)])
def test_camera_frames_prep_on_the_device(net):
    """Camera frames whose source rows do not fit udh_real_prep's shared memory: the kernel reads them from global memory and
    its planes equal cv2.resize(INTER_AREA) of the normalised image bit for bit, for both models' network sizes."""
    from unsuperviseddeephomographyral2018_b200 import _lib, align, dataloader as dl, engine, ops
    rng = np.random.default_rng(net[0])
    I = torch.from_numpy(np.stack([J.textured(rng, 3000, 4000, 3) for _ in range(2)])).cuda()
    _, max_rows = ops.area_table(3000, 4000, net[0], net[1])
    assert _lib.lib.udh_real_prep_smem_bytes(max_rows, 4000) > 227 * 1024
    eng = engine.HomographyEngine(2, 128, net[0], net[1], numeric="fp32", seed=0)
    est = align.HomographyEstimator(engine=eng)
    assert align.prep_path(3000, 4000, *net) == align.PREP_DEVICE
    got = est._planes(I).cpu().numpy()
    for j in range(2):
        host = dl.normalise_resize_host(I[j].cpu().numpy().astype(np.float32), *net)
        assert np.array_equal(_bits(got[j]), _bits(host)), j
