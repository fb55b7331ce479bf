"""GPU tests of the decoder's parallel entropy path (self-synchronising Huffman decode of long segments): with the path
forced on, camera-size files of every sampling, quality, restart layout and kind of content decode bit-identical to
cv2.imread; plans mixing long and short segments, segments that fall back to the serial path after too few
synchronisation rounds, and a truncated long file give what the serial path gives."""
import contextlib

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from oracle import jpeg as J  # noqa: E402

pytestmark = pytest.mark.gpu

SAMPLING = {"4:4:4": 0x111111, "4:2:2": 0x211111, "4:2:0": 0x221111}


def _cv2_rgb(blob):
    return cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)[..., ::-1]


def _content(kind, h, w, rng):
    """smooth: low-frequency gradients; noise: uniform bytes (long codes, frequent FF 00); constant: EOB-only blocks."""
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "constant":
        return np.full((h, w, 3), rng.integers(0, 256, 3), np.uint8)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    f = [np.sin(x / (w / (2 + c)) + y / (h / (3 + c)) + c) for c in range(3)]
    return np.stack([(127.5 + 120 * v).astype(np.uint8) for v in f], axis=2)


def _encode(img, mode, q, rst=0):
    prm = [cv2.IMWRITE_JPEG_QUALITY, q] + ([cv2.IMWRITE_JPEG_RST_INTERVAL, rst] if rst else [])
    if mode == "gray":
        img = img[..., 0]
    else:
        prm += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING[mode]]
    ok, buf = cv2.imencode(".jpg", img, prm)
    assert ok
    return buf.tobytes()


def large_corpus(h, w, seed=0):
    """[(label, bytes)] of one size: every sampling x content at quality 95, quality 30 and 100 at 4:2:0, and 4:2:0 with
    restart intervals of 16 MCUs (segments far below the parallel path's length threshold) and 2000 MCUs (above it)."""
    rng = np.random.default_rng(seed * 7919 + h * 1000 + w)
    imgs = {k: _content(k, h, w, rng) for k in ("smooth", "noise", "constant")}
    out = []
    for kind, img in imgs.items():
        for mode in ("gray", "4:4:4", "4:2:2", "4:2:0"):
            out.append(("%s %s q95" % (kind, mode), _encode(img, mode, 95)))
        for q in (30, 100):
            out.append(("%s 4:2:0 q%d" % (kind, q), _encode(img, "4:2:0", q)))
    for kind in ("smooth", "noise"):
        for rst in (16, 2000):
            out.append(("%s 4:2:0 q95 rst%d" % (kind, rst), _encode(imgs[kind], "4:2:0", 95, rst)))
    return out


@contextlib.contextmanager
def parallel(mode, rounds=16):
    from unsuperviseddeephomographyral2018_b200 import _lib
    _lib.check(_lib.lib.udh_debug_jpeg_set_parallel(mode))
    _lib.check(_lib.lib.udh_debug_jpeg_set_sync_rounds(rounds))
    try:
        yield
    finally:
        _lib.check(_lib.lib.udh_debug_jpeg_set_parallel(-1))
        _lib.check(_lib.lib.udh_debug_jpeg_set_sync_rounds(16))


def _decode(blobs, h, w):
    from unsuperviseddeephomographyral2018_b200 import ops
    plan = ops.JpegPlan(blobs, h, w)
    out, status = plan.decode()
    return out.cpu().numpy(), status.cpu().numpy(), plan


def _has_long_segment(plan):
    from unsuperviseddeephomographyral2018_b200 import _lib
    return _lib.lib.udh_jpeg_plan_workspace_bytes(plan.plan.data_ptr()) > _lib.lib.udh_jpeg_workspace_bytes(plan.n, plan.h, plan.w)


def _parallel_segments(plan):
    """Segments of the last decode that the parallel path decoded (the rest went to the serial path)."""
    import ctypes
    from unsuperviseddeephomographyral2018_b200 import _lib
    n = ctypes.c_int(-1)
    _lib.check(_lib.lib.udh_debug_jpeg_parallel_segments(plan.plan.data_ptr(), ctypes.c_void_p(plan.ws.data_ptr()), ctypes.byref(n)))
    return n.value


def _segments(blob):
    from unsuperviseddeephomographyral2018_b200 import ops
    i = ops.jpeg_parse(blob)
    hm, vm = (i.h_samp[0], i.v_samp[0]) if i.components == 3 else (1, 1)
    nmcu = -(-i.width // (8 * hm)) * -(-i.height // (8 * vm))
    return -(-nmcu // i.restart_interval) if i.restart_interval else 1


@pytest.mark.parametrize("h,w", [(3000, 4000), (2999, 4001), (1080, 1920)])
def test_parallel_path_is_bit_identical_to_cv2(h, w):
    files = large_corpus(h, w)
    with parallel(1):
        for k0 in range(0, len(files), 6):                     # six camera frames per launch keep the workspace small
            chunk = files[k0:k0 + 6]
            got, st, plan = _decode([b for _, b in chunk], h, w)
            assert _has_long_segment(plan)
            # smooth content synchronises; uniform noise and some constant images may not (the serial path decodes those)
            assert _parallel_segments(plan) >= sum(_segments(b) for label, b in chunk if label.startswith("smooth"))
            for k, (label, blob) in enumerate(chunk):
                assert st[k] == 0, label
                assert np.array_equal(got[k], _cv2_rgb(blob)), label


def test_plan_mixing_long_and_short_segments():
    """Length-picked paths (the default): the short files and the restart-interval file stay serial, the long smooth
    frames are decoded by the parallel path, all in one launch."""
    h, w = 1080, 1920
    files = large_corpus(h, w)
    pick = [f for f in files if f[0] in ("constant 4:2:0 q95", "smooth 4:2:0 q100", "smooth 4:2:0 q30", "noise 4:2:0 q95 rst16",
                                          "smooth 4:4:4 q95", "constant gray q95", "noise 4:2:0 q30")]
    assert len(pick) == 7
    lengths = [len(b) for _, b in pick]
    assert min(lengths) < (1 << 17) <= max(lengths)
    got, st, plan = _decode([b for _, b in pick], h, w)
    assert _has_long_segment(plan)
    long_files = sum(len(b) >= (1 << 17) for label, b in pick if "rst" not in label)   # the rst16 file: 7 kB segments
    assert 2 <= _parallel_segments(plan) <= long_files == 3
    assert (st == 0).all()
    for k, (label, blob) in enumerate(pick):
        assert np.array_equal(got[k], _cv2_rgb(blob)), label


@pytest.mark.parametrize("rounds", [0, 1])
def test_too_few_rounds_fall_back_to_the_serial_path(rounds):
    h, w = 1080, 1920
    files = [f for f in large_corpus(h, w) if "4:2:0 q95" in f[0] or "gray" in f[0]]
    with parallel(1, rounds):
        got, st, plan = _decode([b for _, b in files], h, w)
    assert _has_long_segment(plan)
    if rounds == 0:
        assert _parallel_segments(plan) == 0
    assert (st == 0).all()
    for k, (label, blob) in enumerate(files):
        assert np.array_equal(got[k], _cv2_rgb(blob)), label


@pytest.mark.parametrize("mode", [1, -1])
def test_truncated_long_file_gets_the_serial_status(mode):
    from unsuperviseddeephomographyral2018_b200 import _lib
    h, w = 1080, 1920
    files = [b for label, b in large_corpus(h, w) if label in ("smooth 4:2:0 q100", "smooth 4:4:4 q95", "smooth 4:2:2 q95",
                                                                "noise 4:2:0 q30", "smooth 4:2:0 q95 rst2000")]
    cut = len(files[0]) * 2 // 3                                # header intact, entropy data cut short
    blobs = [files[0][:cut]] + files[1:] + [files[0][:len(files[0]) - 3]]   # the last one loses its EOI and a byte
    with parallel(0):
        _, st_serial, _ = _decode(blobs, h, w)
    with parallel(mode):
        got, st, plan = _decode(blobs, h, w)
    assert _has_long_segment(plan)
    assert _parallel_segments(plan) >= 1
    assert st[0] == _lib.JPEG_E["TRUNCATED"]
    assert np.array_equal(st, st_serial)
    for k in range(1, len(blobs) - 1):
        assert st[k] == 0
        assert np.array_equal(got[k], _cv2_rgb(blobs[k])), k


@pytest.mark.parametrize("h,w", J.SIZES)
def test_path_forced_on_and_off_agree_on_the_decoder_corpus(h, w):
    blobs = [b for _, b in J.corpus(h, w)]
    with parallel(1):
        on, st_on, plan = _decode(blobs, h, w)
    assert _has_long_segment(plan)
    with parallel(0):
        off, st_off, plan = _decode(blobs, h, w)
    assert not _has_long_segment(plan)
    assert (st_on == 0).all() and (st_off == 0).all()
    assert np.array_equal(on, off)


def test_path_forced_on_and_off_agree_on_truncated_corpus_files():
    """The existing decoder test's truncations (one segment cut, and a restart-marker file cut) on the parallel path."""
    files = [b for _, b in J.corpus(142, 190)]
    blobs = files[:5] + [files[4][:len(files[4]) * 2 // 3]] + files[6:] + [files[5][:len(files[5]) // 2]]
    res = []
    for mode in (1, 0):
        with parallel(mode):
            got, st, _ = _decode(blobs, 142, 190)
        res.append((got, st))
    assert np.array_equal(res[0][1], res[1][1])
    ok = res[0][1] == 0
    assert ok.sum() == len(blobs) - 2
    assert np.array_equal(res[0][0][ok], res[1][0][ok])


def test_entry_points_reject_bad_switch_values():
    from unsuperviseddeephomographyral2018_b200 import _lib
    assert _lib.lib.udh_debug_jpeg_set_parallel(2) != 0
    assert _lib.lib.udh_debug_jpeg_set_sync_rounds(17) != 0
    assert _lib.lib.udh_jpeg_plan_workspace_bytes(None) == 0
    torch.cuda.synchronize()
