"""CPU tests of the JPEG encoder and the INTER_LINEAR resize: the NumPy restatements (oracle/jpeg_enc.py,
oracle/resize_linear.py) equal cv2 byte for byte / pixel for pixel, the C ABI's capacity matches the restatement's bound
and rejects bad arguments before touching the device, and the new kernels compile for sm_90a without spills."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import jpeg_enc as E  # noqa: E402
from oracle import resize_linear as R  # noqa: E402


def _cv2_encode(img, q):
    ok, buf = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q])
    assert ok
    return buf.tobytes()


@pytest.mark.parametrize("channels", [3, 1])
@pytest.mark.parametrize("h,w", E.SIZES)
def test_encoder_oracle_is_byte_identical_to_cv2(h, w, channels):
    for label, img, q in E.corpus(h, w, channels):
        got = E.encode(img, q)
        assert got == _cv2_encode(img, q), label
        assert len(got) <= E.capacity(h, w, channels), label


def test_corpus_exercises_dummy_blocks_stuffing_and_long_codes():
    """Odd block counts in 4:2:0 (dummy luma blocks right of and below the image), 0xFF bytes to stuff, and quality 100
    noise (the longest AC codes) are all in the corpus."""
    odd = [(h, w) for h, w in E.SIZES if ((h + 7) // 8) % 2 or ((w + 7) // 8) % 2]
    assert {(17, 23), (8, 16), (16, 8), (1, 1)} <= set(odd)
    blob = E.encode(E.image("noise", 240, 320, 3, seed=1), 100)
    assert blob.count(b"\xff\x00") > 1000


def test_headers_depend_only_on_size_channels_and_quality():
    a = E.encode(E.image("noise", 17, 23, 3, seed=1), 75)
    b = E.encode(E.image("zeros", 17, 23, 3), 75)
    hd = E.header(17, 23, 3, 75)
    assert a.startswith(hd) and b.startswith(hd) and len(hd) == 623
    assert len(E.header(17, 23, 1, 75)) == 328


@pytest.mark.parametrize("h,w", [(480, 640), (640, 480), (427, 640), (640, 427), (375, 500), (500, 375), (612, 612),
                                 (150, 200), (200, 150), (240, 320)])
def test_linear_resize_oracle_equals_cv2(h, w):
    img = np.random.default_rng(h * 1000 + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    assert np.array_equal(R.resize_linear(img, 240, 320), cv2.resize(img, (320, 240)))


def test_linear_table_of_the_library_equals_the_oracle():
    from unsuperviseddeephomographyral2018_b200 import ops
    for (h, w, dh, dw) in [(480, 640, 240, 320), (150, 200, 240, 320), (7, 5, 240, 320), (1, 1, 4, 4), (240, 320, 240, 320)]:
        xs, xa0, xa1 = R.column_table(w, dw)
        y0, y1, b0, b1 = R.row_table(h, dh)
        want = np.concatenate([xs, xa0, xa1, y0, b0, b1, y1]).astype(np.int32)
        assert np.array_equal(ops.linear_table(h, w, dh, dw), want), (h, w, dh, dw)


def test_encode_capacity_matches_the_oracle_bound():
    from unsuperviseddeephomographyral2018_b200 import _lib
    L = _lib.lib
    for ch in (1, 3):
        for h, w in E.SIZES + [(65535, 1), (1000, 1001)]:
            assert L.udh_jpeg_encode_capacity(h, w, ch) == E.capacity(h, w, ch), (h, w, ch)
    for bad in ((0, 5, 3), (5, 0, 3), (5, 5, 2), (5, 5, 4), (65536, 5, 3), (-1, 5, 1)):
        assert L.udh_jpeg_encode_capacity(*bad) == 0, bad
    assert L.udh_jpeg_encode_workspace_bytes(0, 8, 8, 3) == 0
    assert L.udh_jpeg_encode_workspace_bytes(2, 8, 8, 2) == 0
    assert L.udh_jpeg_encode_workspace_bytes(2, 8, 8, 3) > 2 * 6 * 64 * 2


def test_encode_entry_rejects_bad_arguments():
    """udh_jpeg_encode checks its arguments before touching the device."""
    from unsuperviseddeephomographyral2018_b200 import _lib
    L = _lib.lib
    p = ctypes.c_void_p(256)                          # never dereferenced: every call below fails its argument checks
    cap = L.udh_jpeg_encode_capacity(17, 23, 3)
    ws = L.udh_jpeg_encode_workspace_bytes(2, 17, 23, 3)
    for i in (0, 6, 8, 9, 10):                        # img, out, nbytes, status, ws
        a = [p, 2, 17, 23, 3, 95, p, cap, p, p, p, ws, None]
        a[i] = None
        assert L.udh_jpeg_encode(*a) == _lib.EINVAL, i
        assert b"udh_jpeg_encode: null pointer" in L.udh_last_error()
    for n, h, w, ch in ((0, 17, 23, 3), (2, 0, 23, 3), (2, 17, 0, 3), (2, 17, 23, 2), (2, 70000, 23, 3)):
        assert L.udh_jpeg_encode(p, n, h, w, ch, 95, p, cap, p, p, p, ws, None) == _lib.EINVAL
        assert b"bad dimensions" in L.udh_last_error()
    for q in (0, 101, -5):
        assert L.udh_jpeg_encode(p, 2, 17, 23, 3, q, p, cap, p, p, p, ws, None) == _lib.EINVAL
        assert b"quality" in L.udh_last_error()
    assert L.udh_jpeg_encode(p, 2, 17, 23, 3, 95, p, cap - 1, p, p, p, ws, None) == _lib.EINVAL
    assert b"below the capacity" in L.udh_last_error()
    assert L.udh_jpeg_encode(p, 2, 17, 23, 3, 95, p, cap, p, p, p, ws - 1, None) == _lib.EWS


def test_linear_resize_entry_rejects_bad_arguments():
    from unsuperviseddeephomographyral2018_b200 import _lib
    L = _lib.lib
    p = ctypes.c_void_p(256)
    for i in (0, 1, 2):
        a = [p, p, p, 1, 480, 640, 240, 320, None]
        a[i] = None
        assert L.udh_resize_linear_u8(*a) == _lib.EINVAL
        assert b"null pointer" in L.udh_last_error()
    for dims in ((-1, 480, 640, 240, 320), (1, 0, 640, 240, 320), (1, 480, 640, 240, 0)):
        assert L.udh_resize_linear_u8(p, p, p, *dims, None) == _lib.EINVAL
        assert b"bad dimensions" in L.udh_last_error()


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return nvcc if os.path.exists(nvcc) else shutil.which("nvcc")


@pytest.mark.skipif(_nvcc() is None, reason="nvcc is not installed")
@pytest.mark.parametrize("src,kernels", [("jpeg_enc.cu", ["enc_coef_kernel", "enc_scan_kernel", "enc_write_kernel", "enc_stuff_kernel"]),
                                         ("real_prep.cu", ["resize_up_u8_kernelILb1E"])])
def test_new_kernels_compile_for_sm90a_without_spills(tmp_path, src, kernels):
    from unsuperviseddeephomographyral2018_b200 import build_ext
    cmd = [_nvcc()] + build_ext.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build_ext.CSRC, src), "-o", str(tmp_path / "k.o")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout
    report, current = {}, None
    for line in out.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            current = m.group(1)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            report[current] = tuple(int(v) for v in m.groups())
    assert "sm_90a" in out
    for k in kernels:
        found = [v for name, v in report.items() if k in name]
        assert found, "ptxas -v printed no report for %s" % k
        for stack, st, ld in found:
            assert stack == 0 and st == 0 and ld == 0, (k, stack, st, ld)
