"""CPU tests of the PNG decoder: the NumPy / zlib restatement (oracle/png.py) against cv2 bit for bit, the chunks both
skip, and the library's host parser and plan through the C ABI (what they accept, what they report, and why they reject)."""
import os
import re
import shutil
import struct
import subprocess
import zlib

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import png as PNG  # noqa: E402


def _cv2(blob):
    return cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)


@pytest.mark.parametrize("h,w", PNG.SIZES)
def test_oracle_is_bit_identical_to_cv2(h, w):
    files = PNG.corpus(h, w)
    assert len(files) == 3 * 11 + 1
    for label, blob in files:
        got, ref = PNG.decode(blob), _cv2(blob)
        assert got.shape == ref.shape == (h, w, 3), label
        assert np.array_equal(got, ref), label


def test_cv2_writes_every_block_type():
    """Level 0 writes stored blocks, level 1 fixed or dynamic ones, levels 6 and 9 dynamic ones: the corpus covers all three."""
    img = PNG.textured(np.random.default_rng(5), 64, 50, 3)
    kinds = set()
    for label, blob in PNG.corpus(64, 50):
        stream = PNG.parse(blob)[2]
        kinds.add((stream[2] >> 1) & 3)          # BTYPE of the first block
    assert kinds >= {0, 1, 2} or kinds >= {0, 2}
    assert (PNG.parse(cv2.imencode(".png", img, [cv2.IMWRITE_PNG_COMPRESSION, 0])[1].tobytes())[2][2] >> 1) & 3 == 0
    flat = PNG.make_png(np.zeros((4, 5, 3), np.uint8), [0] * 4, level=1)
    assert (PNG.parse(flat)[2][2] >> 1) & 3 == 1


def test_every_filter_type_is_exercised():
    for label, blob in PNG.corpus(17, 23):
        if label.startswith("zlib-c3-f"):
            raw = zlib.decompress(PNG.parse(blob)[2])
            f = int(label[-1])
            assert {raw[y * (1 + 23 * 3)] for y in range(17)} == {f}, label


def _ancillary(typ):
    body = {b"tEXt": b"Comment\x00made by a test", b"zTXt": b"Comment\x00\x00" + zlib.compress(b"compressed text"),
            b"iTXt": b"Comment\x00\x00\x00en\x00\x00international text", b"tIME": struct.pack(">HBBBBB", 2024, 5, 6, 7, 8, 9),
            b"pHYs": struct.pack(">IIB", 3780, 3780, 1), b"gAMA": struct.pack(">I", 100000), b"sBIT": bytes([5, 6, 5]),
            b"tRNS": struct.pack(">HHH", 1, 2, 3), b"sRGB": bytes([0]), b"eXIf": b"MM\x00\x2a\x00\x00\x00\x08\x00\x00"}[typ]
    return PNG.chunk(typ, body)


def test_ignored_chunks_do_not_change_what_cv2_returns():
    from unsuperviseddeephomographyral2018_b200 import ops
    px = PNG.textured(np.random.default_rng(3), 19, 21, 3)
    plain = PNG.make_png(px, [4] * 19)
    ref = _cv2(plain)
    for typ in PNG.IGNORED:
        blob = PNG.make_png(px, [4] * 19, extra=[_ancillary(typ)])
        assert np.array_equal(_cv2(blob), ref), typ
        assert np.array_equal(PNG.decode(blob), ref), typ
        assert ops.png_parse(blob).reason == 0, typ
    every = PNG.make_png(px, [4] * 19, extra=[_ancillary(t) for t in PNG.IGNORED])
    assert np.array_equal(_cv2(every), ref) and ops.png_parse(every).reason == 0


def test_other_ancillary_chunks_go_to_the_host():
    from unsuperviseddeephomographyral2018_b200 import _lib, ops
    px = PNG.textured(np.random.default_rng(4), 9, 10, 3)
    for typ in (b"gAMA", b"sBIT", b"tRNS", b"sRGB", b"eXIf"):
        blob = PNG.make_png(px, [0] * 9, extra=[_ancillary(typ)])
        assert ops.png_parse(blob).reason == _lib.PNG_R["CHUNK"] == PNG.parse(blob)[0], typ


def test_parser_reports_size_depth_and_colour_type():
    from unsuperviseddeephomographyral2018_b200 import ops
    img = PNG.textured(np.random.default_rng(0), 31, 45, 3)
    for src, ct, ch in ((img[..., 0], 0, 1), (img, 2, 3), (np.concatenate([img, img[..., :1]], axis=2), 6, 4)):
        blob = cv2.imencode(".png", src)[1].tobytes()
        info = ops.png_parse(blob)
        assert (info.reason, info.height, info.width, info.bit_depth, info.color_type, info.interlace, info.channels) == (0, 31, 45, 8, ct, 0, ch)
        assert info.idat_bytes == len(PNG.parse(blob)[2])


def _palette_png():
    h, w = 5, 6
    raw = b"".join(b"\x00" + bytes(range(w)) for _ in range(h))
    plte = PNG.chunk(b"PLTE", bytes(range(3 * w)))
    return PNG.SIG + PNG.ihdr(h, w, 8, 3) + plte + PNG.chunk(b"IDAT", zlib.compress(raw)) + PNG.chunk(b"IEND", b"")


def _interlaced_png():
    """An Adam7 header in front of a non-interlaced stream: the parser rejects it on the header alone."""
    px = PNG.textured(np.random.default_rng(6), 8, 8, 3)
    blob = PNG.make_png(px, [0] * 8)
    return PNG.SIG + PNG.ihdr(8, 8, 8, 2, 1) + blob[8 + 25:]


def test_parser_gives_a_distinct_reason_for_each_unsupported_file():
    from unsuperviseddeephomographyral2018_b200 import _lib, ops
    img = PNG.textured(np.random.default_rng(1), 24, 30, 3)
    plain = cv2.imencode(".png", img)[1].tobytes()
    n_idat = PNG.SIG.__len__() + 25 + 8                      # the first IDAT payload byte (cv2 writes IHDR then IDAT)
    assert plain[n_idat - 4:n_idat] == b"IDAT"
    bad_crc = bytearray(plain)
    bad_crc[n_idat + 5] ^= 0x10
    sub8 = PNG.SIG + PNG.ihdr(4, 4, 4, 0) + PNG.chunk(b"IDAT", zlib.compress(b"\x00\x00\x00" * 4)) + PNG.chunk(b"IEND", b"")
    files = {
        "PALETTE": _palette_png(),
        "DEPTH16": cv2.imencode(".png", img.astype(np.uint16) * 257)[1].tobytes(),
        "DEPTH_SUB8": sub8,
        "INTERLACED": _interlaced_png(),
        "CRC": bytes(bad_crc),
        "IDAT_TRUNCATED": plain[:n_idat + 20],
        "NO_IEND": plain[:-12],
        "NOT_PNG": b"GIF89a" + bytes(40),
        "JPEG": cv2.imencode(".jpg", img)[1].tobytes(),
        "TRUNCATED": plain[:8 + 10],
    }
    reasons = {k: ops.png_parse(b).reason for k, b in files.items()}
    assert reasons == {k: _lib.PNG_R[k] for k in files}
    assert len(set(reasons.values())) == len(files)
    assert {k: PNG.parse(b)[0] for k, b in files.items()} == reasons          # the oracle's parser agrees
    assert ops.png_parse(plain).reason == 0
    assert ops.png_parse(b"").reason == _lib.PNG_R["NOT_PNG"]
    # cv2 reads the palette and 16-bit files: they are valid PNGs the host decoder takes
    for k in ("PALETTE", "DEPTH16"):
        assert _cv2(files[k]) is not None, k


def test_plan_refuses_unsupported_and_wrong_size_files():
    from unsuperviseddeephomographyral2018_b200 import _lib, ops
    img = PNG.textured(np.random.default_rng(2), 17, 23, 3)
    good = cv2.imencode(".png", img)[1].tobytes()
    gray = cv2.imencode(".png", img[..., 0])[1].tobytes()
    plan = ops.PngPlan([good, gray, good], 17, 23)
    assert plan.idat.numel() == 2 * len(PNG.parse(good)[2]) + len(PNG.parse(gray)[2])
    idat = plan.idat.numpy().tobytes()
    assert idat.startswith(PNG.parse(good)[2] + PNG.parse(gray)[2])
    with pytest.raises(_lib.UdhError, match="image 1 is not supported"):
        ops.PngPlan([good, cv2.imencode(".png", img.astype(np.uint16))[1].tobytes()], 17, 23)
    with pytest.raises(_lib.UdhError, match="image 0 is not supported"):
        ops.PngPlan([cv2.imencode(".jpg", img)[1].tobytes()], 17, 23)
    with pytest.raises(_lib.UdhError, match="image 0 is 17x23"):
        ops.PngPlan([good], 18, 23)


@pytest.mark.skipif(shutil.which(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")) is None, reason="needs nvcc")
def test_png_kernels_do_not_spill(tmp_path):
    from unsuperviseddeephomographyral2018_b200 import build_ext
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    src = os.path.join(build_ext.CSRC, "png.cu")
    out = subprocess.run([nvcc] + build_ext.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "png.o")],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    entries = re.split(r"Compiling entry function", out.stdout + out.stderr)
    kernels = [e for e in entries if "png_inflate_kernel" in e.split("\n")[0] or "png_unfilter_kernel" in e.split("\n")[0]]
    assert len(kernels) == 2
    for e in kernels:
        assert re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", e), e
