"""CPU tests of the baseline-JPEG decoder: the NumPy restatement (oracle/jpeg.py) against cv2 bit for bit, and the
library's host parser through the C ABI (what it accepts, what it reports, and why it rejects)."""
import os
import re
import shutil
import struct
import subprocess

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import jpeg as J  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cv2_rgb(blob):
    return cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)[..., ::-1]


@pytest.mark.parametrize("h,w", J.SIZES)
def test_oracle_is_bit_identical_to_cv2(h, w):
    for label, blob in J.corpus(h, w):
        got, ref = J.decode(blob), _cv2_rgb(blob)
        assert got.shape == ref.shape == (h, w, 3), label
        assert np.array_equal(got, ref), label


def _encode(img, *prm):
    ok, buf = cv2.imencode(".png" if prm == ("png",) else ".jpg", img, [] if prm == ("png",) else list(prm))
    assert ok
    return buf.tobytes()


def _with_exif_orientation(blob, orientation):
    tiff = b"MM\x00\x2a\x00\x00\x00\x08" + struct.pack(">H", 1) + struct.pack(">HHIHH", 0x0112, 3, 1, orientation, 0) + b"\x00" * 4
    app1 = b"Exif\x00\x00" + tiff
    return blob[:2] + b"\xff\xe1" + struct.pack(">H", len(app1) + 2) + app1 + blob[2:]


def test_parser_reports_size_sampling_and_restart_interval():
    from unsuperviseddeephomographyral2018_b200 import ops
    img = J.textured(np.random.default_rng(0), 142, 190, 3)
    for samp, hv in [(0x111111, (1, 1)), (0x211111, (2, 1)), (0x221111, (2, 2))]:
        for ri in (0, 1, 7):
            info = ops.jpeg_parse(_encode(img, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp, cv2.IMWRITE_JPEG_RST_INTERVAL, ri))
            assert info.reason == 0
            assert (info.height, info.width, info.components) == (142, 190, 3)
            assert (info.h_samp[0], info.v_samp[0]) == hv
            assert [info.h_samp[1], info.v_samp[1], info.h_samp[2], info.v_samp[2]] == [1, 1, 1, 1]
            assert info.restart_interval == ri
    info = ops.jpeg_parse(_encode(img[..., 0], cv2.IMWRITE_JPEG_OPTIMIZE, 1))
    assert (info.reason, info.height, info.width, info.components) == (0, 142, 190, 1)


def test_parser_gives_a_distinct_reason_for_each_unsupported_file():
    from unsuperviseddeephomographyral2018_b200 import _lib, ops
    img = J.textured(np.random.default_rng(1), 64, 48, 3)
    plain = _encode(img)
    files = {
        "NOT_BASELINE": _encode(img, cv2.IMWRITE_JPEG_PROGRESSIVE, 1),
        "SAMPLING_H": _encode(img, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x411111),
        "SAMPLING_V": _encode(img, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x121111),
        "ORIENTATION": _with_exif_orientation(plain, 6),
        "NOT_JPEG": _encode(img, "png"),
        "TRUNCATED": plain[:100],
    }
    reasons = {k: ops.jpeg_parse(b).reason for k, b in files.items()}
    assert reasons == {k: _lib.JPEG_R[k] for k in files}
    assert len(set(reasons.values())) == len(files)
    assert ops.jpeg_parse(_with_exif_orientation(plain, 1)).reason == 0
    assert ops.jpeg_parse(b"").reason == _lib.JPEG_R["NOT_JPEG"]
    # the oracle parses what the library parses, and cv2 agrees the file is a plain JPEG
    assert J.decode(_with_exif_orientation(plain, 1)).shape == (64, 48, 3)


def test_plan_refuses_unsupported_and_wrong_size_files():
    from unsuperviseddeephomographyral2018_b200 import _lib, ops
    img = J.textured(np.random.default_rng(2), 17, 23, 3)
    good = _encode(img, cv2.IMWRITE_JPEG_RST_INTERVAL, 1)
    ops.JpegPlan([good, good], 17, 23)
    with pytest.raises(_lib.UdhError, match="image 1 is not supported"):
        ops.JpegPlan([good, _encode(img, cv2.IMWRITE_JPEG_PROGRESSIVE, 1)], 17, 23)
    with pytest.raises(_lib.UdhError, match="image 0 is 17x23"):
        ops.JpegPlan([good], 18, 23)


@pytest.mark.skipif(shutil.which(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")) is None, reason="needs nvcc")
def test_entropy_kernel_does_not_spill(tmp_path):
    from unsuperviseddeephomographyral2018_b200 import build_ext
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    src = os.path.join(build_ext.CSRC, "jpeg.cu")
    out = subprocess.run([nvcc] + build_ext.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "jpeg.o")],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    log = out.stdout + out.stderr
    entries = re.split(r"Compiling entry function", log)
    kernels = [e for e in entries if "jpeg_entropy_kernel" in e.split("\n")[0]]
    assert len(kernels) == 2
    for e in kernels:
        assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", e), e


def _with_dht(blob, tc_th, counts, vals):
    """blob with one more DHT segment right after SOI (parsed before the file's own tables)."""
    body = bytes([tc_th]) + bytes(counts) + bytes(vals)
    return blob[:2] + b"\xff\xc4" + struct.pack(">H", len(body) + 2) + body + blob[2:]


@pytest.mark.parametrize("tc_th,counts", [
    (0x10, [255] + [0] * 15),             # over-subscribed: 255 codes of length 1 (would index past the lookahead table)
    (0x10, [3] + [0] * 15),               # over-subscribed by one
    (0x10, [2] + [0] * 15),               # complete code: the all-ones codeword '1' is used
    (0x11, [0, 2, 3] + [1] * 12 + [2]),   # all-ones codeword at length 16
    (0x00, [0, 1] + [0] * 14),            # DC symbol 16 > 15
])
def test_parser_rejects_malformed_huffman_tables(tc_th, counts):
    from unsuperviseddeephomographyral2018_b200 import _lib, ops
    plain = _encode(J.textured(np.random.default_rng(4), 32, 32, 3))
    vals = [16] if tc_th == 0x00 else [k % 256 for k in range(sum(counts))]
    assert ops.jpeg_parse(_with_dht(plain, tc_th, counts, vals)).reason == _lib.JPEG_R["TRUNCATED"]
    # well-formed extra tables (later redefined by the file's own) are accepted; the second one stops one code short of
    # the all-ones codeword at length 16
    assert ops.jpeg_parse(_with_dht(plain, tc_th, [1, 1] + [0] * 14, [1, 2])).reason == 0
    if tc_th != 0x00:
        ok_counts = [0, 2, 3] + [1] * 13
        assert ops.jpeg_parse(_with_dht(plain, tc_th, ok_counts, list(range(sum(ok_counts))))).reason == 0
