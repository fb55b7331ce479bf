"""GPU tests of the PNG decoder: bit-identical to cv2 on the fixture set (one launch per size, and 1024 images in one
launch), every malformed-stream path ending in a per-image status without a fault, and the on-disk loaders (plain and
real-data) giving the same batches from PNG and mixed JPEG + PNG sets as with every file read by cv2.imread."""
import os
import zlib

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from oracle import png as PNG  # noqa: E402

pytestmark = pytest.mark.gpu


def _cv2(blob):
    return cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)


@pytest.mark.parametrize("h,w", PNG.SIZES + [(240, 320)])
def test_device_decode_is_bit_identical_to_cv2(h, w):
    from unsuperviseddeephomographyral2018_b200 import ops
    files = PNG.corpus(h, w)
    out, status = ops.decode_png([b for _, b in files], h, w)                # one launch mixes every variant of this size
    rgb, _ = ops.decode_png([b for _, b in files], h, w, rgb=True)
    assert status.cpu().eq(0).all()
    got, got_rgb = out.cpu().numpy(), rgb.cpu().numpy()
    for k, (label, blob) in enumerate(files):
        ref = _cv2(blob)
        assert np.array_equal(got[k], ref), label
        assert np.array_equal(got_rgb[k], ref[..., ::-1]), label


def test_1024_images_in_one_launch():
    from unsuperviseddeephomographyral2018_b200 import ops
    rng = np.random.default_rng(11)
    h, w = 48, 70
    blobs = []
    for k in range(1024):
        c = (1, 3, 4)[k % 3]
        img = PNG.textured(rng, h, w, 3)
        src = img[..., 0] if c == 1 else (np.concatenate([img, img[..., :1]], axis=2) if c == 4 else img)
        prm = [cv2.IMWRITE_PNG_COMPRESSION, int(rng.integers(0, 10))]
        if k % 5 == 0:
            prm += [cv2.IMWRITE_PNG_STRATEGY, cv2.IMWRITE_PNG_STRATEGY_DEFAULT]
        blobs.append(cv2.imencode(".png", src, prm)[1].tobytes())
    out, status = ops.decode_png(blobs, h, w)
    assert status.cpu().eq(0).all()
    got = out.cpu().numpy()
    for k, blob in enumerate(blobs):
        assert np.array_equal(got[k], _cv2(blob)), k


class _Bits:
    """LSB-first deflate bit writer (Huffman codes are written most significant bit first)."""

    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, value, nbits):
        self.v |= value << self.n
        self.n += nbits

    def code(self, code, nbits):
        self.put(int(format(code, "0%db" % nbits)[::-1], 2), nbits)

    def bytes(self):
        return self.v.to_bytes((self.n + 7) // 8, "little")


def _fixed_block(tokens):
    """One final fixed-Huffman block: tokens are literal byte values or (length, distance code, distance extra bits)
    with length 3 (code 257)."""
    b = _Bits()
    b.put(1, 1); b.put(1, 2)
    for t in tokens:
        if isinstance(t, int):
            b.code(0x30 + t, 8) if t < 144 else b.code(0x190 + t - 144, 9)
        else:
            b.code(1, 7)                                   # symbol 257: length 3
            b.code(t[1], 5)
    b.code(0, 7)                                           # end of block
    return b.bytes()


def _zlib(deflate, raw):
    return b"\x78\x01" + deflate + zlib.adler32(raw).to_bytes(4, "big")


def _corrupt_files(h=6, w=7):
    """(label, file, expected status or None for any nonzero status, pixels) -- every file parses; its stream is bad."""
    from unsuperviseddeephomographyral2018_b200 import _lib
    rng = np.random.default_rng(9)
    px = PNG.textured(rng, h, w, 3)[..., ::-1]
    raw = PNG.filter_rows(px, [4] * h)
    good = zlib.compress(raw, 9)
    E = _lib.PNG_E
    flipped = bytearray(good)
    flipped[len(good) // 2] ^= 0x08
    bad_filter = bytearray(raw)
    bad_filter[(1 + 3 * w) * 2] = 5
    far = _zlib(_fixed_block([(3, 0, 0)] + [0] * (len(raw) - 3)), raw)      # a match at position 0: distance 1 > 0 bytes out
    return [
        ("huffman-bit", PNG.make_png(px, None, stream=bytes(flipped)), None),
        ("distance", PNG.make_png(px, None, stream=far), E["DISTANCE"]),
        ("adler", PNG.make_png(px, None, stream=good[:-4] + bytes(4)), E["ADLER"]),
        ("short", PNG.make_png(px, None, stream=zlib.compress(raw[:-5])), E["SHORT"]),
        ("long", PNG.make_png(px, None, stream=zlib.compress(raw + bytes(5))), E["LONG"]),
        ("filter", PNG.make_png(px, None, stream=zlib.compress(bytes(bad_filter))), E["FILTER"]),
        ("truncated", PNG.make_png(px, None, stream=good[:len(good) // 2]), E["TRUNCATED"]),
        ("zlib-header", PNG.make_png(px, None, stream=b"\x79" + good[1:]), E["ZLIB"]),
        ("block-type-3", PNG.make_png(px, None, stream=b"\x78\x01\x07" + good[3:]), E["BLOCK"]),
    ], px


def test_corrupt_streams_end_in_a_status_and_the_others_decode():
    from unsuperviseddeephomographyral2018_b200 import _lib, ops
    bad, px = _corrupt_files()
    h, w = px.shape[:2]
    good = [PNG.make_png(px, [f] * h) for f in range(5)]
    blobs = []
    for k, (_, blob, _) in enumerate(bad):
        blobs += [good[k % 5], blob]
    for _, blob, _ in bad:
        assert ops.png_parse(blob).reason == 0
    out, status = ops.PngPlan(blobs, h, w).decode()
    torch.cuda.synchronize()                                                 # the launch itself reports no error
    st = status.cpu().numpy()
    got = out.cpu().numpy()
    for k, (label, blob, expect) in enumerate(bad):
        assert st[2 * k] == 0 and np.array_equal(got[2 * k], _cv2(good[k % 5])), label
        assert st[2 * k + 1] != 0, label
        if expect is not None:
            assert st[2 * k + 1] == expect, (label, st[2 * k + 1])
    with pytest.raises(_lib.UdhError, match="image 1 failed"):
        ops.decode_png(blobs, h, w)


# ---- the loaders --------------------------------------------------------------------------------------------------------
def _write(path, img, kind, rng):
    if kind == "png":
        prm = [cv2.IMWRITE_PNG_COMPRESSION, int(rng.integers(0, 10))]
    elif kind == "png-long":       # parses, fails on the device (more image data than rows); libpng warns and reads it
        raw_img = img if img.ndim == 3 else img[..., None]
        px = raw_img[..., ::-1] if raw_img.shape[2] == 3 else raw_img
        blob = PNG.make_png(px, None, stream=zlib.compress(PNG.filter_rows(px, [1] * px.shape[0]) + bytes(5)))
        with open(path, "wb") as f:
            f.write(blob)
        return
    elif kind == "png16":
        img = img.astype(np.uint16) * 257
        prm = []
    else:
        prm = [cv2.IMWRITE_JPEG_QUALITY, 95]
    assert cv2.imwrite(path, img, prm)


def _write_set(root, kinds, sizes, n=20, P=128, rho=4, seed=0, net=(240, 320)):
    """The reference's on-disk layout with pair i written as kinds[i % len(kinds)] at sizes[i % len(sizes)], gray on a third
    of the files."""
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "I")); os.makedirs(os.path.join(root, "I_prime"))
    names, pts1, gt = [], [], []
    for i in range(n):
        name = "%06d.%s" % (i + 1, "jpg" if kinds[i % len(kinds)] == "jpg" else "png")
        for sub in ("I", "I_prime"):
            gray = (i + (sub == "I")) % 3 == 0
            hh, ww = sizes[i % len(sizes)]
            img = PNG.textured(rng, hh, ww, 3)
            _write(os.path.join(root, sub, name), img[..., 0] if gray else img, kinds[i % len(kinds)], rng)
        names.append("%s %s" % (name, name))
        x0, y0 = rng.integers(rho, net[1] - rho - P), rng.integers(rho, net[0] - rho - P)
        pts1.append([x0, y0, x0 + P, y0, x0 + P, y0 + P, x0, y0 + P])
        gt.append(rng.integers(-rho, rho + 1, 8))
    with open(os.path.join(root, "list.txt"), "w") as f:
        f.write("\n".join(names) + "\n")
    np.savetxt(os.path.join(root, "pts1.txt"), np.array(pts1, np.float64))
    np.savetxt(os.path.join(root, "gt.txt"), np.array(gt, np.float64))


def _force_host_decode(m):
    """Make both parsers reject every file: the loader then decodes all of them with cv2.imread."""
    from unsuperviseddeephomographyral2018_b200 import _lib, ops

    def reject_jpeg(blob):
        info = _lib.JpegInfo(); info.reason = _lib.JPEG_R["NOT_JPEG"]
        return info

    def reject_png(blob):
        info = _lib.PngInfo(); info.reason = _lib.PNG_R["NOT_PNG"]
        return info
    m.setattr(ops, "jpeg_parse", reject_jpeg)
    m.setattr(ops, "png_parse", reject_png)


def _plain_batches(root, mode, nb, monkeypatch, host):
    from unsuperviseddeephomographyral2018_b200 import dataloader
    with monkeypatch.context() as m:
        if host:
            _force_host_decode(m)
        prm = dataloader.dataloader_params(data_path=str(root), filenames_file=os.path.join(root, "list.txt"),
                                           pts1_file=os.path.join(root, "pts1.txt"), gt_file=os.path.join(root, "gt.txt"), mode=mode,
                                           batch_size=8, img_h=240, img_w=320, patch_size=128, augment_list=["normalize"], do_augment=0.5)
        dl = dataloader.Dataloader(prm, shuffle=True, seed=3)
        out = [{k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in dl.next_batch().items()} for _ in range(nb)]
        torch.cuda.synchronize()
    return out, dict(dl.decode_stats)


def _same(dev, ref):
    assert len(dev) == len(ref)
    for k in range(len(ref)):
        assert dev[k].keys() == ref[k].keys()
        for key, v in ref[k].items():
            if isinstance(v, torch.Tensor):
                assert torch.equal(dev[k][key], v), (k, key)
            elif isinstance(v, np.ndarray):
                assert np.array_equal(dev[k][key], v), (k, key)
            else:
                assert v is None and dev[k][key] is None, (k, key)


@pytest.mark.parametrize("mode", ["train", "test"])
def test_png_set_batches_match_the_host_decoder(tmp_path, monkeypatch, mode):
    # mostly PNG; one pair in eleven a wrong size, one a 16-bit PNG (host), one a stream that fails on the device
    kinds = ["png"] * 8 + ["png16", "png", "png-long"]
    _write_set(tmp_path, kinds, [(240, 320)] * 6 + [(120, 160)])
    nb = 7                                                                   # 56 pairs of a 20-pair set: two epoch boundaries
    dev, st = _plain_batches(tmp_path, mode, nb, monkeypatch, host=False)
    ref, ref_st = _plain_batches(tmp_path, mode, nb, monkeypatch, host=True)
    _same(dev, ref)
    assert st["png_images"] > 0 and st["png_images"] == st["device_images"] and st["decode_errors"] >= 1 and st["host_images"] > 0
    assert ref_st["device_images"] == 0


def test_mixed_jpeg_and_png_set_batches_match_the_host_decoder(tmp_path, monkeypatch):
    _write_set(tmp_path, ["png", "jpg", "png", "jpg", "jpg"], [(240, 320)])
    dev, st = _plain_batches(tmp_path, "test", 5, monkeypatch, host=False)
    ref, _ = _plain_batches(tmp_path, "test", 5, monkeypatch, host=True)
    _same(dev, ref)
    assert 0 < st["png_images"] < st["device_images"] and st["host_images"] == 0


def _real_loader(root, mode, do_augment, B):
    from unsuperviseddeephomographyral2018_b200 import dataloader as dl
    prm = dl.extended_dataloader_params(data_path=str(root), filenames_file=os.path.join(root, "list.txt"),
                                        pts1_file=os.path.join(root, "pts1.txt"), gt_file=os.path.join(root, "gt.txt"),
                                        mode=mode, batch_size=B, img_h=142, img_w=190, patch_size=128, augment_list=["normalize"],
                                        do_augment=do_augment, full_img_h=240, full_img_w=320)
    return dl.Dataloader(prm, shuffle=True, seed=7, device="cuda")


@pytest.mark.parametrize("mode,do_augment", [("train", 0.5), ("test", 1.0)])
def test_real_data_loader_takes_png_at_both_sizes(tmp_path, mode, do_augment):
    """Full-size and network-size PNG files (gray and colour, some JPEG) through the real-data loader: the same batches as
    its host path."""
    _write_set(tmp_path, ["png", "png", "jpg", "png"], [(240, 320), (142, 190), (240, 320)], net=(142, 190))
    dev, host = _real_loader(tmp_path, mode, do_augment, 8), _real_loader(tmp_path, mode, do_augment, 8)
    assert dev._extended_on_device() and (142, 190) in dev._decode_sizes()
    nb = 4
    got = [{k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in dev.next_batch().items()} for _ in range(nb)]
    ref = [{k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in host._disk_batch_extended_host().items()} for _ in range(nb)]
    _same(got, ref)
    st = dev.decode_stats
    assert st["png_images"] > 0 and st["png_images"] < st["device_images"] and st["host_images"] == 0
