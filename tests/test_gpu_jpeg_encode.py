"""GPU tests of the baseline-JPEG encoder and the INTER_LINEAR resize: device files byte-identical to cv2.imencode on the
seeded corpus at 1, 7 and 300 images per launch, the device decoder reading them back as cv2 does, and the device resize
equal to cv2.resize on a batch of mixed source sizes."""
import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from oracle import jpeg_enc as E  # noqa: E402

pytestmark = pytest.mark.gpu


def _cv2_encode(img, q):
    ok, buf = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q])
    assert ok
    return buf.tobytes()


@pytest.mark.parametrize("channels", [3, 1])
@pytest.mark.parametrize("h,w", E.SIZES)
def test_device_encode_is_byte_identical_to_cv2_one_per_launch(h, w, channels):
    from unsuperviseddeephomographyral2018_b200 import ops
    for label, img, q in E.corpus(h, w, channels):
        got = ops.encode_jpeg(img[None], quality=q)
        assert len(got) == 1 and got[0] == _cv2_encode(img, q), label


@pytest.mark.parametrize("channels", [3, 1])
@pytest.mark.parametrize("h,w", E.SIZES)
def test_device_encode_is_byte_identical_to_cv2_seven_per_launch(h, w, channels):
    from unsuperviseddeephomographyral2018_b200 import ops
    imgs = [img for _, img, q in E.corpus(h, w, channels) if q == 95] + [E.image("noise", h, w, channels, seed=7)]
    assert len(imgs) == 7
    for q in (10, 95, 100):
        got = ops.encode_jpeg(torch.from_numpy(np.stack(imgs)).cuda(), quality=q)
        for k, img in enumerate(imgs):
            assert got[k] == _cv2_encode(img, q), (k, q)


@pytest.mark.parametrize("h,w,channels", [(240, 320, 3), (240, 320, 1), (17, 23, 3)])
def test_device_encode_is_byte_identical_to_cv2_three_hundred_per_launch(h, w, channels):
    from unsuperviseddeephomographyral2018_b200 import ops
    imgs = np.stack([E.image(E.KINDS[k % len(E.KINDS)], h, w, channels, seed=k) for k in range(300)])
    got = ops.encode_jpeg(imgs, quality=95)
    assert len(got) == 300
    for k in range(300):
        assert got[k] == _cv2_encode(imgs[k], 95), k


def test_device_decoder_reads_device_encoded_files_as_cv2_does():
    from unsuperviseddeephomographyral2018_b200 import ops
    for h, w in ((240, 320), (17, 23), (9, 9)):
        for channels in (3, 1):
            imgs = np.stack([E.image(k, h, w, channels, seed=3) for k in E.KINDS])
            blobs = ops.encode_jpeg(imgs, quality=90)
            out, status = ops.decode_jpeg(blobs, h, w)
            got = out.cpu().numpy()
            for k, blob in enumerate(blobs):
                want = cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)[..., ::-1]
                assert np.array_equal(got[k], want), (h, w, channels, k)


def test_encode_rejects_bad_input_shapes():
    from unsuperviseddeephomographyral2018_b200 import _lib, ops
    with pytest.raises(_lib.UdhError, match="BGR"):
        ops.encode_jpeg(np.zeros((2, 8, 8, 4), np.uint8))
    with pytest.raises(_lib.UdhError, match="quality"):
        ops.encode_jpeg(np.zeros((2, 8, 8, 3), np.uint8), quality=0)


def test_device_linear_resize_equals_cv2_on_mixed_sizes():
    from unsuperviseddeephomographyral2018_b200 import ops
    rng = np.random.default_rng(5)
    sizes = [(480, 640), (427, 640), (640, 427), (375, 500), (612, 612), (150, 200), (240, 320), (480, 640), (375, 500)]
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]
    groups = {}
    for k, im in enumerate(imgs):
        groups.setdefault(im.shape, []).append(k)
    for shape, ks in groups.items():                                  # one launch per source size
        out = ops.resize_linear_u8(torch.from_numpy(np.stack([imgs[k] for k in ks])).cuda(), 240, 320).cpu().numpy()
        for j, k in enumerate(ks):
            assert np.array_equal(out[j], cv2.resize(imgs[k], (320, 240))), shape
    small = rng.integers(0, 256, (3, 7, 5, 3), dtype=np.uint8)
    out = ops.resize_linear_u8(torch.from_numpy(small).cuda(), 33, 2).cpu().numpy()
    for j in range(3):
        assert np.array_equal(out[j], cv2.resize(small[j], (2, 33)))
