"""CPU tests of the real-data generator (gen_real_data.py) with the host backend: draws, names, text files, labels and
cutoffs equal a transcription of the reference's homographyGeneration / dataCollection in train and test mode; the
files are cv2.imencode of cv2.resize(cv2.imread(frame)); --debug, --resume and gray files behave as the module states;
and the repository's real-data Dataloader reads the generated test set."""
import os

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")
sio = pytest.importorskip("scipy.io")

from oracle import gen_real_data as OR  # noqa: E402

# flags scaled to small frames so that randint(rho, img_w - rho - patch_size) has a range
SMALL = ["--img_h", "40", "--img_w", "60", "--full_img_h", "48", "--full_img_w", "64", "--patch_size", "16", "--rho", "4"]


def write_frames(root, ids, seed=0):
    """Overlapping frames DSC_<id>.JPG of a panning camera, plus files the *.JPG glob must not take."""
    rng = np.random.default_rng(seed)
    os.makedirs(root, exist_ok=True)
    scene = np.clip(rng.normal(128, 50, (90, 200, 3)), 0, 255).astype(np.uint8)
    scene = cv2.GaussianBlur(scene, (5, 5), 0)
    for k, i in enumerate(ids):
        cv2.imwrite(os.path.join(root, "DSC_%04d.JPG" % i), scene[:, 6 * k:6 * k + 120])
    cv2.imwrite(os.path.join(root, "DSC_9999.jpg"), scene[:, :120])
    cv2.imwrite(os.path.join(root, "DSC_9998.png"), scene[:, :120])
    return root


def write_labels(root, nframes, seed=1, split=12):
    rng = np.random.default_rng(seed)
    c1 = rng.uniform(0, 640, (4 * nframes, 2))
    c2 = c1 + rng.uniform(-20, 20, c1.shape)
    os.makedirs(root, exist_ok=True)
    files = [os.path.join(root, "a.mat"), os.path.join(root, "b.mat")]
    sio.savemat(files[0], {"all_corr1": c1[:split], "all_corr2": c2[:split]})
    sio.savemat(files[1], {"all_corr1": c1[split:], "all_corr2": c2[split:]})
    return files, c1, c2


def args_for(tmp, mode, extra=(), num_data=7, test_num_data=5, im_per_im=3):
    from unsuperviseddeephomographyral2018_b200 import gen_real_data as G
    argv = ["--mode", mode, "--raw_data_path", str(tmp / "train"), "--test_raw_data_path", str(tmp / "test"),
            "--data_path", str(tmp / "data") + "/", "--num_data", str(num_data), "--test_num_data", str(test_num_data),
            "--im_per_im", str(im_per_im)] + SMALL + list(extra)
    return G.resolve_args(G.build_parser().parse_args(argv))


def _savetxt(rows):
    return "".join("%s\n" % " ".join("%.18e" % v for v in r) for r in rows)


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def _host_file(frame, size, gray=False):
    im = cv2.resize(cv2.imread(frame), (size[1], size[0]))
    if gray:
        im = cv2.cvtColor(im, cv2.COLOR_RGB2GRAY)
    return cv2.imencode(".jpg", im, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes()


def _check_set(args, d, want, gray=False):
    for n, I_file, Ip_file, _, _ in want:
        name = "%d.jpg" % n
        assert _read(os.path.join(d, "I", name)) == _host_file(I_file, (40, 60), gray)
        assert _read(os.path.join(d, "FULL_I", name)) == _host_file(I_file, (48, 64), gray)
        assert _read(os.path.join(d, "I_prime", name)) == _host_file(Ip_file, (40, 60), gray)
        assert _read(os.path.join(d, "FULL_I_prime", name)) == _host_file(Ip_file, (48, 64), gray)
    for sub in ("I", "FULL_I", "I_prime", "FULL_I_prime"):
        assert sorted(os.listdir(os.path.join(d, sub))) == sorted("%d.jpg" % n for n, *_ in want)


@pytest.mark.parametrize("num_data,im_per_im", [(7, 3), (20, 4), (2, 3)])
def test_train_mode_follows_the_reference(tmp_path, num_data, im_per_im):
    from unsuperviseddeephomographyral2018_b200 import gen_real_data as G
    write_frames(tmp_path / "train", [57, 58, 59, 60, 61, 62])      # pairs 59 and 60 are on the train ignore list
    args = args_for(tmp_path, "train", num_data=num_data, im_per_im=im_per_im)
    end = G.generate(args, OR.HostBackend(), seed=3)
    nxt, want = OR.reference_samples(str(tmp_path / "train"), G.TRAIN_IGNORE, num_data, 0, im_per_im, 4, 16, 40, seed=3, width=60)
    assert end == nxt == len(want) == min(num_data, 3 * im_per_im)
    assert [os.path.basename(w[1]) for w in want][::im_per_im] == ["DSC_0057.JPG", "DSC_0058.JPG", "DSC_0061.JPG"][:len(want[::im_per_im])]
    d = str(tmp_path / "data")
    assert _read(os.path.join(d, "pts1.txt")).decode() == _savetxt(w[3] for w in want)
    assert _read(os.path.join(d, "train_real.txt")).decode() == "".join("%d.jpg %d.jpg\n" % (n, n) for n, *_ in want)
    assert not os.path.exists(os.path.join(d, "gt.txt")) and not os.path.exists(os.path.join(d, "test_gt.txt"))
    _check_set(args, d, want)


def test_cutoff_in_the_middle_of_a_pair(tmp_path):
    from unsuperviseddeephomographyral2018_b200 import gen_real_data as G
    write_frames(tmp_path / "train", [1, 2, 3, 4])
    end = G.generate(args_for(tmp_path, "train", num_data=5, im_per_im=3), OR.HostBackend(), seed=0)
    assert end == 5
    d = str(tmp_path / "data")
    assert len(_read(os.path.join(d, "pts1.txt")).splitlines()) == 5
    assert _read(os.path.join(d, "I_prime", "4.jpg")) == _host_file(str(tmp_path / "train" / "DSC_0003.JPG"), (40, 60))


def test_test_mode_reads_the_labels_and_follows_the_reference(tmp_path):
    from unsuperviseddeephomographyral2018_b200 import dataloader, gen_real_data as G
    ids = [28, 29, 30, 31, 32, 33]                                   # pairs 30 and 31 are on the test ignore list
    write_frames(tmp_path / "test", ids, seed=4)
    files, c1, c2 = write_labels(tmp_path / "labels", len(ids) - 1)
    args = args_for(tmp_path, "test", extra=["--test_labels"] + files, num_data=100, test_num_data=8, im_per_im=2)
    assert args.start_index == 100 and args.num_data == 8
    end = G.generate(args, OR.HostBackend(), seed=9)
    nxt, want = OR.reference_samples(str(tmp_path / "test"), G.TEST_IGNORE, 8, 100, 2, 4, 16, 40, corr=(c1, c2), seed=9, width=60)
    assert end == nxt == 106 and len(want) == 6
    d = str(tmp_path / "data")
    assert _read(os.path.join(d, "test_pts1.txt")).decode() == _savetxt(w[3] for w in want)
    assert _read(os.path.join(d, "test_gt.txt")).decode() == _savetxt(w[4] for w in want)
    assert _read(os.path.join(d, "test_real.txt")).decode() == "".join("%d.jpg %d.jpg\n" % (n, n) for n, *_ in want)
    # the last accepted pair is frame position 4 (id 32): rows 16..19, counted over the ignored pairs too
    assert np.array_equal(want[-1][4], np.hstack([c1[16:20].flatten(), c2[16:20].flatten()]))
    _check_set(args, d, want)
    # the repository's real-data loader reads the set (host path); gt rows are the 16 correspondence numbers
    p = dataloader.extended_dataloader_params(data_path=d + "/", filenames_file=os.path.join(d, "test_real.txt"),
                                              pts1_file=os.path.join(d, "test_pts1.txt"), gt_file=os.path.join(d, "test_gt.txt"),
                                              mode="test", batch_size=3, img_h=40, img_w=60, patch_size=16, augment_list=[],
                                              do_augment=0.0, full_img_h=48, full_img_w=64)
    dl = dataloader.Dataloader(p, shuffle=False, device="cpu")
    b = dl._disk_batch_extended_host()
    assert b["gt_corr"].shape == (3, 16)
    assert np.array_equal(b["gt_corr"], np.array([w[4] for w in want[:3]], np.float32))
    assert np.array_equal(b["pts1"].numpy(), np.array([w[3] for w in want[:3]]))


def test_default_labels_are_the_reference_files(tmp_path):
    args = args_for(tmp_path, "test")
    from unsuperviseddeephomographyral2018_b200 import gen_real_data as G
    assert args.test_labels == [os.path.join(str(tmp_path / "test"), "labels", f) for f in G.LABEL_FILES]
    assert args.ignore_list == [30, 31] and args_for(tmp_path, "train").ignore_list == G.TRAIN_IGNORE


def test_debug_draws_one_sample_and_writes_nothing(tmp_path):
    from unsuperviseddeephomographyral2018_b200 import gen_real_data as G
    write_frames(tmp_path / "train", [59, 60, 61, 62])
    end = G.generate(args_for(tmp_path, "train", extra=["--debug", "true"]), OR.HostBackend(), seed=0)
    assert end == 1
    assert os.listdir(tmp_path / "data") == []
    nxt, _ = OR.reference_samples(str(tmp_path / "train"), G.TRAIN_IGNORE, 7, 0, 3, 4, 16, 40, debug=True)
    assert nxt == end


def test_resume_deletes_only_when_gt_file_exists(tmp_path):
    """--resume N removes gt_file first; the real generator never writes it, so nothing is deleted unless the user put
    one there, and FULL_I* are never deleted.  The text files are opened 'wb' on every run, --resume Y included."""
    from unsuperviseddeephomographyral2018_b200 import gen_real_data as G
    write_frames(tmp_path / "train", [1, 2, 3, 4])
    d = tmp_path / "data"
    G.generate(args_for(tmp_path, "train", num_data=6, im_per_im=2), OR.HostBackend(), seed=0)
    G.generate(args_for(tmp_path, "train", num_data=2, im_per_im=2), OR.HostBackend(), seed=1)
    assert sorted(os.listdir(d / "I")) == ["%d.jpg" % i for i in range(6)]
    assert len(_read(str(d / "pts1.txt")).splitlines()) == 2
    G.generate(args_for(tmp_path, "train", extra=["--resume", "Y", "--start_index", "6"], num_data=1, im_per_im=2), OR.HostBackend(), seed=2)
    assert _read(str(d / "train_real.txt")) == b"6.jpg 6.jpg\n"
    (d / "gt.txt").write_bytes(b"")
    G.generate(args_for(tmp_path, "train", num_data=2, im_per_im=2), OR.HostBackend(), seed=3)
    assert not (d / "gt.txt").exists()
    assert sorted(os.listdir(d / "I")) == ["0.jpg", "1.jpg"] and sorted(os.listdir(d / "I_prime")) == ["0.jpg", "1.jpg"]
    assert sorted(os.listdir(d / "FULL_I")) == ["%d.jpg" % i for i in range(7)]


def test_train_without_color_writes_gray_files(tmp_path):
    from unsuperviseddeephomographyral2018_b200 import gen_real_data as G
    write_frames(tmp_path / "train", [1, 2, 3])
    args = args_for(tmp_path, "train", extra=["--color", "false"], num_data=3, im_per_im=2)
    G.generate(args, OR.HostBackend(), seed=0)
    _, want = OR.reference_samples(str(tmp_path / "train"), G.TRAIN_IGNORE, 3, 0, 2, 4, 16, 40, seed=0, width=60)
    _check_set(args, str(tmp_path / "data"), want, gray=True)
    assert cv2.imread(str(tmp_path / "data" / "FULL_I" / "0.jpg"), cv2.IMREAD_UNCHANGED).ndim == 2
