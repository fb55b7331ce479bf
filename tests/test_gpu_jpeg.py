"""GPU tests of the baseline-JPEG decoder: bit-identical to cv2 on the seeded corpus, per-image failure without a fault,
the on-disk Dataloader giving the same batches with the device decoder as with the host one, and the two CLIs that read
the on-disk test set giving the same results either way."""
import os

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from oracle import jpeg as J  # noqa: E402

pytestmark = pytest.mark.gpu


def _cv2_rgb(blob):
    return cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)[..., ::-1]


@pytest.mark.parametrize("lanes", [32, 1])
@pytest.mark.parametrize("h,w", J.SIZES)
def test_device_decode_is_bit_identical_to_cv2(h, w, lanes):
    from unsuperviseddeephomographyral2018_b200 import _lib, ops
    files = J.corpus(h, w)
    _lib.check(_lib.lib.udh_debug_jpeg_set_lanes(lanes))
    try:
        out, status = ops.decode_jpeg([b for _, b in files], h, w)          # one launch mixes every variant of this size
    finally:
        _lib.check(_lib.lib.udh_debug_jpeg_set_lanes(32))
    assert status.cpu().eq(0).all()
    got = out.cpu().numpy()
    for k, (label, blob) in enumerate(files):
        assert np.array_equal(got[k], _cv2_rgb(blob)), label


def test_truncated_entropy_data_fails_only_that_image():
    from unsuperviseddeephomographyral2018_b200 import _lib, ops
    corpus = J.corpus(142, 190)
    assert corpus[5][0].endswith("rst1") and corpus[1][0].endswith("rst1") and corpus[4][0].endswith("plain")
    files = [b for _, b in corpus]
    cut = files[4][:len(files[4]) * 2 // 3]      # header intact, entropy data cut short: one segment (no restart markers)
    cut_rst = files[5][:len(files[5]) // 2]      # the same in a file with a restart marker after every MCU
    blobs = files[:5] + [cut] + files[6:] + [cut_rst]
    plan = ops.JpegPlan(blobs, 142, 190)
    out, status = plan.decode()
    torch.cuda.synchronize()                                                 # the launch itself reports no error
    st = status.cpu().numpy()
    assert st[5] == _lib.JPEG_E["TRUNCATED"] and st[-1] == _lib.JPEG_E["TRUNCATED"]
    assert (np.delete(st, [5, len(st) - 1]) == 0).all()
    got = out.cpu().numpy()
    for k, blob in enumerate(blobs):
        if k not in (5, len(blobs) - 1):
            assert np.array_equal(got[k], _cv2_rgb(blob)), k
    with pytest.raises(_lib.UdhError, match="image 5 failed"):
        ops.decode_jpeg(blobs, 142, 190)


def _write_dataset(root, n=20, h=240, w=320, P=128, rho=32, seed=0, truncate=None):
    """The reference's on-disk layout (I/, I_prime/, list, pts1.txt, gt.txt, and the same lists under the test_* names the
    CLIs read): mixed gray and colour files, restart markers on some, one progressive pair and one wrong-size pair (host
    fallback).  truncate = i cuts pair i's I' file in its entropy-coded data."""
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "I")); os.makedirs(os.path.join(root, "I_prime"))
    names, pts1, gt = [], [], []
    for i in range(n):
        name = "%06d.jpg" % (i + 1)
        for sub in ("I", "I_prime"):
            gray = (i + (sub == "I")) % 3 == 0
            hh, ww = (120, 160) if i == 7 else (h, w)
            img = J.textured(rng, hh, ww, 1 if gray else 3)
            prm = [cv2.IMWRITE_JPEG_QUALITY, 95]
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
        x0, y0 = rng.integers(rho, w - rho - P), rng.integers(rho, h - rho - P)
        pts1.append([x0, y0, x0 + P, y0, x0 + P, y0 + P, x0, y0 + P])
        gt.append(rng.integers(-rho, rho + 1, 8))
    with open(os.path.join(root, "list.txt"), "w") as f:
        f.write("\n".join(names) + "\n")
    np.savetxt(os.path.join(root, "pts1.txt"), np.array(pts1, np.float64))
    np.savetxt(os.path.join(root, "gt.txt"), np.array(gt, np.float64))
    for a, b in (("list.txt", "test_synthetic.txt"), ("pts1.txt", "test_pts1.txt"), ("gt.txt", "test_gt.txt")):
        with open(os.path.join(root, a)) as f, open(os.path.join(root, b), "w") as g:
            g.write(f.read())


def _force_host_decode(m):
    """Make the parser reject every file: the loader then decodes all of them with cv2.imread."""
    from unsuperviseddeephomographyral2018_b200 import _lib, ops

    def reject(blob):
        info = _lib.JpegInfo(); info.reason = _lib.JPEG_R["NOT_JPEG"]
        return info
    m.setattr(ops, "jpeg_parse", reject)


def _batches(root, mode, nb, monkeypatch, host):
    from unsuperviseddeephomographyral2018_b200 import dataloader, ops
    calls = []
    with monkeypatch.context() as m:
        if host:
            _force_host_decode(m)
        real = ops.JpegPlan.decode
        m.setattr(ops.JpegPlan, "decode", lambda self, device=None: calls.append(self.n) or real(self, device))
        prm = dataloader.dataloader_params(data_path=str(root), filenames_file=os.path.join(root, "list.txt"),
                                           pts1_file=os.path.join(root, "pts1.txt"), gt_file=os.path.join(root, "gt.txt"), mode=mode,
                                           batch_size=8, img_h=240, img_w=320, patch_size=128, augment_list=["normalize"], do_augment=0.5)
        dl = dataloader.Dataloader(prm, shuffle=True, seed=3)
        out = [{k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in dl.next_batch().items()} for _ in range(nb)]
        torch.cuda.synchronize()
    return out, calls, dict(dl.decode_stats)


@pytest.mark.parametrize("mode", ["train", "test"])
def test_disk_loader_batches_match_the_host_decoder(tmp_path, monkeypatch, mode):
    _write_dataset(tmp_path)
    nb = 7                                                                  # 56 pairs of a 20-pair set: two epoch boundaries
    dev, calls, _ = _batches(tmp_path, mode, nb, monkeypatch, host=False)
    ref, ref_calls, _ = _batches(tmp_path, mode, nb, monkeypatch, host=True)
    assert calls and sum(calls) > 0 and not ref_calls
    for k in range(nb):
        assert dev[k].keys() == ref[k].keys()
        for key, v in ref[k].items():
            if isinstance(v, torch.Tensor):
                assert torch.equal(dev[k][key], v), (k, key)
            else:
                assert v is None and dev[k][key] is None, (k, key)


def test_device_decode_errors_go_to_the_host_decoder(tmp_path, monkeypatch):
    """A file whose entropy data is cut short passes the parser and fails on the device (nonzero status); the loader hands
    it to cv2.imread, which decodes what is there ("Premature end of JPEG file"), so the batches still equal the host's."""
    _write_dataset(tmp_path, truncate=3)
    dev, _, st = _batches(tmp_path, "test", 3, monkeypatch, host=False)
    ref, _, ref_st = _batches(tmp_path, "test", 3, monkeypatch, host=True)
    assert st["decode_errors"] >= 1 and ref_st["decode_errors"] == 0 and st["device_images"] > 0
    for k in range(3):
        for key, v in ref[k].items():
            if isinstance(v, torch.Tensor):
                assert torch.equal(dev[k][key], v), (k, key)


def _run_cli(script, argv, capsys, monkeypatch, host):
    """Run a CLI's main() in this process (host=True: every file through cv2.imread) -> its stdout."""
    import importlib
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    monkeypatch.syspath_prepend(root)
    mod = importlib.import_module(script)
    with monkeypatch.context() as m:
        if host:
            _force_host_decode(m)
        capsys.readouterr()
        rc = mod.main(argv)
        out = capsys.readouterr().out
    assert rc in (0, None), out[-2000:]
    sys.stdout.flush()
    return out


def _without_times(text):
    """Printed lines with the timing fields removed (they are wall-clock measurements, not results)."""
    import re
    out = []
    for ln in text.splitlines():
        if ln.startswith("Running time:"):
            continue
        ln = re.sub(r", time [0-9.e+-]+", "", ln)
        if ln.startswith("output_line:"):
            ln = ln.rsplit(",", 1)[0]
        out.append(ln)
    return out


def test_conventional_direct_method_gives_the_same_results_with_either_decoder(tmp_path, monkeypatch, capsys):
    _write_dataset(tmp_path / "data")
    res = []
    for host in (False, True):
        log = tmp_path / ("log_host" if host else "log_dev")
        argv = ["--method", "direct", "--mode", "test", "--data_path", str(tmp_path / "data") + "/", "--log_dir", str(log),
                "--batch_size", "8", "--num_gpus", "1"]
        out = _run_cli("homography_conventional_synthetic", argv, capsys, monkeypatch, host)
        (path,) = [os.path.join(d, f) for d, _, fs in os.walk(log) for f in fs if f == "results.txt"]
        with open(path) as f:
            numbers = f.read().split()
        res.append((numbers[:4], _without_times(out)))          # the fifth number is seconds per sample
    assert res[0][0] == res[1][0]
    assert [ln for ln in res[0][1] if "log_dev" not in ln] == [ln for ln in res[1][1] if "log_host" not in ln]
    assert any(ln.startswith(" Test| image") for ln in res[0][1])


def test_cnn_test_mode_gives_the_same_metrics_with_either_decoder(tmp_path, monkeypatch, capsys):
    _write_dataset(tmp_path / "data")
    outs = []
    for host in (False, True):
        argv = ["--mode", "test", "--data_path", str(tmp_path / "data") + "/", "--batch_size", "8", "--num_gpus", "1",
                "--numeric", "bf16x3", "--do_augment", "0.5", "--model_dir", str(tmp_path / "m"), "--log_dir", str(tmp_path / "l"),
                "--results_dir", str(tmp_path / "r")]
        out = _run_cli("homography_CNN_synthetic", argv, capsys, monkeypatch, host)
        lines = out.splitlines()
        i = next(k for k, ln in enumerate(lines) if ln.startswith("|Steps"))
        outs.append(lines[i:i + 4])                              # the metrics line and the percentiles
    assert outs[0] == outs[1]
    assert len(outs[0][1].split()) == 4
