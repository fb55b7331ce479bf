"""GPU tests of gen_real_data.py: on camera-size frames (device decode, parallel entropy path) plus a progressive and an
EXIF-rotated frame (host fallback), the device generator writes a directory byte-identical to the host generator's in
train mode with and without colour and in test mode with labels; homography_CNN_real.py --mode test then runs on the
generated test set through the device loader, prints its metrics and writes its report images."""
import importlib
import os
import sys

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")
sio = pytest.importorskip("scipy.io")

from oracle import gen_real_data as OR  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W = 3000, 4000


def with_orientation(blob, orientation):
    """blob with an EXIF APP1 (big-endian TIFF, IFD0 holding only the orientation tag) right after SOI."""
    be = lambda v, n: v.to_bytes(n, "big")
    tiff = b"MM\x00\x2a" + be(8, 4) + be(1, 2) + be(0x0112, 2) + be(3, 2) + be(1, 4) + be(orientation, 2) + b"\0\0" + be(0, 4)
    payload = b"Exif\x00\x00" + tiff
    return blob[:2] + b"\xff\xe1" + be(len(payload) + 2, 2) + payload + blob[2:]


def write_sequence(root, ids, seed=0):
    """Overlapping 12 MP frames of a panning camera, quality 95 4:2:0 (baseline, one entropy segment of several MB);
    the third is progressive and the fifth carries EXIF orientation 6 (both are used by accepted pairs)."""
    rng = np.random.default_rng(seed)
    os.makedirs(root, exist_ok=True)
    small = rng.integers(0, 256, (H // 40, (W + 200 * len(ids)) // 40, 3), dtype=np.uint8)
    scene = cv2.resize(small, (small.shape[1] * 40, small.shape[0] * 40), interpolation=cv2.INTER_CUBIC)
    scene = cv2.add(scene, rng.integers(0, 24, scene.shape, dtype=np.uint8))
    for k, i in enumerate(ids):
        img = np.ascontiguousarray(scene[:, 200 * k:200 * k + W])
        prm = [cv2.IMWRITE_JPEG_QUALITY, 95] + ([cv2.IMWRITE_JPEG_PROGRESSIVE, 1] if k == 2 else [])
        blob = cv2.imencode(".jpg", img, prm)[1].tobytes()
        if k == 4:
            blob = with_orientation(blob, 6)
        with open(os.path.join(root, "DSC_%04d.JPG" % i), "wb") as f:
            f.write(blob)
    return root


@pytest.fixture(scope="module")
def frames(tmp_path_factory):
    root = tmp_path_factory.mktemp("frames")
    write_sequence(str(root / "train"), [57, 58, 59, 60, 61, 62, 63])
    write_sequence(str(root / "test"), [28, 29, 30, 31, 32, 33, 34], seed=1)
    rng = np.random.default_rng(2)
    c1 = rng.uniform(0, 640, (24, 2))
    os.makedirs(root / "test" / "labels")
    labels = []
    for k, (a, b) in enumerate(((0, 12), (12, 24))):
        labels.append(str(root / "test" / "labels" / ("c%d.mat" % k)))
        sio.savemat(labels[-1], {"all_corr1": c1[a:b], "all_corr2": c1[a:b] + 3.5})
    return root, labels


def _tree(d):
    out = {}
    for base, _, files in os.walk(d):
        for f in files:
            p = os.path.join(base, f)
            with open(p, "rb") as fh:
                out[os.path.relpath(p, d)] = fh.read()
    return out


def _run(root, data, mode, backend, extra=()):
    from unsuperviseddeephomographyral2018_b200 import gen_real_data as G
    argv = ["--mode", mode, "--raw_data_path", str(root / "train"), "--test_raw_data_path", str(root / "test"),
            "--data_path", data + "/", "--im_per_im", "3", "--num_data", "40", "--test_num_data", "11"] + list(extra)
    args = G.resolve_args(G.build_parser().parse_args(argv))
    return G.generate(args, backend, seed=7)


@pytest.mark.parametrize("mode,extra", [("train", ()), ("train", ("--color", "false")), ("test", None)],
                         ids=["train-colour", "train-gray", "test-labels"])
def test_device_directory_equals_the_host_directory(frames, tmp_path, monkeypatch, mode, extra):
    from unsuperviseddeephomographyral2018_b200 import _lib, gen_real_data as G, ops
    root, labels = frames
    extra = ("--test_labels",) + tuple(labels) if extra is None else extra
    raw = root / ("train" if mode == "train" else "test")
    reasons = [ops.jpeg_parse(open(os.path.join(raw, f), "rb").read()).reason for f in sorted(os.listdir(raw)) if f.endswith(".JPG")]
    assert reasons == [0, 0, _lib.JPEG_R["NOT_BASELINE"], 0, _lib.JPEG_R["ORIENTATION"], 0, 0]
    host_reads = []
    real_read = G.read_frame
    monkeypatch.setattr(G, "read_frame", lambda p: host_reads.append(os.path.basename(p)) or real_read(p))
    n_dev = _run(root, str(tmp_path / "dev"), mode, G.DeviceBackend(), extra)
    monkeypatch.undo()
    n_host = _run(root, str(tmp_path / "host"), mode, OR.HostBackend(), extra)
    assert n_dev == n_host
    names = sorted(n for n in os.listdir(raw) if n.endswith(".JPG"))
    assert sorted(host_reads) == [names[2], names[4]]
    dev, host = _tree(str(tmp_path / "dev")), _tree(str(tmp_path / "host"))
    assert sorted(dev) == sorted(host)
    bad = [k for k in host if dev[k] != host[k]]
    assert not bad, bad[:5]
    samples = n_dev - (40 if mode == "test" else 0)
    assert sum(k.startswith("FULL_I_prime") for k in dev) == samples == (11 if mode == "test" else 12)


def test_cnn_real_test_mode_runs_on_the_generated_set(frames, tmp_path, monkeypatch, capsys):
    from unsuperviseddeephomographyral2018_b200 import dataloader, gen_real_data as G
    root, labels = frames
    data = str(tmp_path / "data")
    _run(root, data, "test", G.DeviceBackend(), ("--test_labels",) + tuple(labels))
    monkeypatch.syspath_prepend(ROOT)
    mod = importlib.import_module("homography_CNN_real")
    def host_path(self):
        raise AssertionError("the generated set must take the device loader")
    monkeypatch.setattr(dataloader.Dataloader, "_disk_batch_extended_host", host_path)
    argv = ["--mode", "test", "--data_path", data + "/", "--batch_size", "4", "--num_gpus", "1", "--load_model_dir", str(tmp_path / "m"),
            "--save_model_dir", str(tmp_path / "s"), "--log_dir", str(tmp_path / "l"), "--results_dir", str(tmp_path / "r")]
    capsys.readouterr()
    rc = mod.main(argv)
    out = capsys.readouterr().out
    sys.stdout.flush()
    assert rc in (0, None), out[-2000:]
    assert any(ln.startswith("|Steps") for ln in out.splitlines()), out[-2000:]
    images = [f for _, _, fs in os.walk(tmp_path / "r") for f in fs if f.endswith(".jpg")]
    assert len(images) >= 8
