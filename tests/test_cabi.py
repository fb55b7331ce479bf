"""CPU tests of the drop-in boundary: libudh.so builds/loads, exports every symbol include/udh.h declares, keeps
the Python and C parameter layouts identical, and fails loudly (no CPU fallback) when there is no GPU."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "udh.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(udh_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from unsuperviseddeephomographyral2018_b200 import _lib
    syms = declared_symbols()
    assert len(syms) >= 19
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for s in syms:
        assert hasattr(raw, s), "libudh.so does not export %s" % s
    assert sorted(_lib.SIGNATURES) == syms, "ctypes table and include/udh.h disagree"
    assert _lib.lib.udh_version() >= 100
    assert isinstance(_lib.lib.udh_last_error(), bytes)


def test_parameter_layout_matches_between_python_and_c():
    from unsuperviseddeephomographyral2018_b200 import _lib, params
    specs = params.param_specs(128)
    assert params.num_parameters(specs) == 34192264                      # SURVEY §8a row C
    assert _lib.lib.udh_param_total_floats(128) == params.total_floats(specs)
    for i, s in enumerate(specs.values()):
        off, n = ctypes.c_size_t(), ctypes.c_size_t()
        assert _lib.lib.udh_param_offset(128, i, ctypes.byref(off), ctypes.byref(n)) == 0
        assert (off.value, n.value) == (s.offset, s.size), s.name
        assert s.offset % 32 == 0
    assert _lib.lib.udh_param_offset(128, 20, ctypes.byref(off), ctypes.byref(n)) == _lib.EINVAL
    assert b"bad tensor index" in _lib.lib.udh_last_error()
    assert _lib.lib.udh_cnn_workspace_bytes(128, 128, 0) > 128 * 13_000_000   # ~13.2 MB of activations per pair
    assert _lib.lib.udh_cnn_workspace_bytes(4, 100, 0) == 0                   # unsupported patch size


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback_without_a_gpu():
    from unsuperviseddeephomographyral2018_b200 import _lib, engine, ops
    assert _lib.lib.udh_device_available() == 0
    with pytest.raises(_lib.UdhError):
        _lib.require_device()
    with pytest.raises(_lib.UdhError):
        engine.HomographyEngine(2)
    with pytest.raises(_lib.UdhError):
        ops.dlt_forward(torch.zeros(1, 8), torch.zeros(1, 8))


def test_x3_mask_and_row_tile_debug_entries_reject_bad_arguments():
    """udh_debug_x3_conv_ex / udh_debug_x3_conv_rows are exported and check their arguments before touching the device."""
    from unsuperviseddeephomographyral2018_b200 import _lib
    L = _lib.lib
    raw = ctypes.CDLL(_lib.LIB_PATH)
    assert hasattr(raw, "udh_debug_x3_conv_ex") and hasattr(raw, "udh_debug_x3_conv_rows")
    p = ctypes.c_void_p(256)                          # never dereferenced: every call below fails its argument checks
    for i in (0, 1, 5, 6):                            # x, w, out, scratch
        a = [p, p, None, None, None, p, p]
        a[i] = None
        assert L.udh_debug_x3_conv_ex(*a, 2, 16, 16, 64, 64, 1, 0, None) == _lib.EINVAL
        assert b"udh_debug_x3_conv_ex: null pointer" in L.udh_last_error()
    for i in (0, 1, 4, 6):                            # x, w, out, scratch
        a = [p, p, p, None, p, p, p]
        a[i] = None
        assert L.udh_debug_x3_conv_rows(*a, 2, 16, 128, 1, None) == _lib.EINVAL
        assert b"udh_debug_x3_conv_rows: null pointer" in L.udh_last_error()
    assert L.udh_debug_x3_conv_rows(p, p, None, None, p, p, p, 2, 16, 128, 1, None) == _lib.EINVAL      # pooled forward: no bias
    assert L.udh_debug_x3_conv_rows(p, p, p, None, p, None, p, 2, 16, 128, 1, None) == _lib.EINVAL      # pooled forward: no codes
    assert L.udh_debug_x3_conv_rows(p, p, p, None, p, p, p, 2, 16, 128, 3, None) == _lib.EINVAL        # rows must be 1 or 2
    assert L.udh_debug_x3_conv_rows(p, p, None, None, p, None, p, 2, 16, 64, 2, None) == _lib.EINVAL    # W != 128
    assert L.udh_debug_x3_conv_rows(p, p, None, None, p, None, p, 2, 15, 128, 2, None) == _lib.EINVAL   # odd height
    assert b"udh_debug_x3_conv_rows" in L.udh_last_error()


def test_mosaic_blends_reject_bad_optional_inputs_before_touching_the_device():
    """udh_mosaic_blend_u8 / udh_mosaic_multiband_u8 check gains, maps, masks, rois and the workspace before their first
    CUDA call: every rejection below names its problem and returns before any device pointer is used."""
    from unsuperviseddeephomographyral2018_b200 import _lib
    L = _lib.lib
    p = ctypes.c_void_p(256)                          # never dereferenced: every call below fails its argument checks
    n, H, W = 2, 8, 8
    frames = (ctypes.c_void_p * n)(256, 512)
    sizes = (ctypes.c_int32 * (2 * n))(4, 4, 4, 4)
    rois = (ctypes.c_int32 * (4 * n))(0, 0, 4, 4, 2, 2, 6, 6)
    masks = (ctypes.c_void_p * n)(256, 512)
    null_mask = (ctypes.c_void_p * n)(256, None)
    maps = (_lib.GainMap * n)(*[_lib.GainMap(256, 256, 256, 2, 2, 1, 0)] * n)
    bad_maps = (_lib.GainMap * n)(_lib.GainMap(256, 256, 256, 2, 2, 1, 0), _lib.GainMap(256, 256, 256, 0, 2, 1, 0))
    cases = [(p, maps, None, rois, "gains and maps exclude each other"), (None, None, masks, None, "masks and maps need rois"),
             (None, maps, None, None, "masks and maps need rois"), (None, None, null_mask, rois, "frame 1's mask is a null pointer"),
             (None, bad_maps, None, rois, "frame 1's gain map is malformed")]
    nb = L.udh_mosaic_workspace_bytes(n)
    for gains, mp, mk, rr, msg in cases:
        assert L.udh_mosaic_blend_u8(frames, sizes, p, gains, mp, mk, rr, n, 3, p, p, H, W, 4, p, p, p, nb, None) == _lib.EINVAL, msg
        assert ("udh_mosaic_blend_u8: " + msg).encode() in L.udh_last_error()
    assert L.udh_mosaic_blend_u8(frames, sizes, p, None, maps, masks, rois, n, 3, p, p, H, W, 4, p, p, p, nb - 1, None) == _lib.EWS
    assert b"udh_mosaic_blend_u8: workspace of" in L.udh_last_error()
    nb = L.udh_mosaic_multiband_workspace_bytes(rois, n, H, W, 2)
    assert nb > 0
    for gains, mp, mk, rr, msg in cases:
        if rr is None:
            msg = "null pointer"                      # the multi-band blend always takes rois
        assert L.udh_mosaic_multiband_u8(frames, sizes, p, gains, mp, mk, rr, n, 3, H, W, 2, p, p, p, nb, None) == _lib.EINVAL, msg
        assert ("udh_mosaic_multiband_u8: " + msg).encode() in L.udh_last_error()
    assert L.udh_mosaic_multiband_u8(frames, sizes, p, None, maps, masks, rois, n, 3, H, W, 2, p, p, p, nb - 1, None) == _lib.EWS
    assert b"udh_mosaic_multiband_u8: workspace of" in L.udh_last_error()


def test_tc_pool_debug_entry_rejects_bad_arguments():
    """udh_debug_tc_pool is exported and checks its arguments before touching the device."""
    from unsuperviseddeephomographyral2018_b200 import _lib
    L = _lib.lib
    assert hasattr(ctypes.CDLL(_lib.LIB_PATH), "udh_debug_tc_pool")
    p = ctypes.c_void_p(256)                          # never dereferenced: every call below fails its argument checks
    for mode in (_lib.NUMERIC_FP32, -1, 3):
        assert L.udh_debug_tc_pool(mode, p, p, p, p, p, 2, 16, 16, 64, None) == _lib.EINVAL
        assert b"unknown numeric_mode" in L.udh_last_error()
    for mode in (_lib.NUMERIC_BF16, _lib.NUMERIC_BF16X3):
        # (in, out, codes, dout, din): no direction, forward without out, no codes, backward without dout
        for a in ((None, p, p, p, None), (p, None, p, None, None), (p, p, None, None, None), (None, None, p, None, p)):
            assert L.udh_debug_tc_pool(mode, *a, 2, 16, 16, 64, None) == _lib.EINVAL, (mode, a)
            assert b"udh_debug_tc_pool: null pointer" in L.udh_last_error()
        for B, H, W, C in ((0, 16, 16, 64), (2, 15, 16, 64), (2, 16, 7, 64), (2, 16, 16, 4), (2, 0, 16, 64)):
            assert L.udh_debug_tc_pool(mode, p, p, p, p, p, B, H, W, C, None) == _lib.EINVAL, (B, H, W, C)
            assert b"udh_debug_tc_pool: needs" in L.udh_last_error()


def test_x3_conv1_mask_debug_entry_rejects_bad_arguments():
    """udh_debug_x3_conv1_ex is exported and checks its arguments before touching the device."""
    from unsuperviseddeephomographyral2018_b200 import _lib
    L = _lib.lib
    p = ctypes.c_void_p(256)                          # never dereferenced: every call below fails its argument checks
    # (I1, I2, w, bias, mask_out, out, g, dW, db, scratch)
    for a, msg in (((None, p, p, p, p, p, None, None, None, p), b"null pointer"),
                   ((p, p, p, p, p, p, None, None, None, None), b"null pointer"),
                   ((p, p, p, p, None, None, None, None, None, p), b"null pointer"),
                   ((p, p, None, p, None, p, None, None, None, p), b"forward needs weights and bias"),
                   ((p, p, None, None, p, None, p, p, p, p), b"mask_out needs the forward"),
                   ((p, p, None, None, None, None, p, None, p, p), b"wgrad needs dW and db")):
        assert L.udh_debug_x3_conv1_ex(*a, 2, 16, 128, None) == _lib.EINVAL, a
        assert b"udh_debug_x3_conv1_ex: " + msg in L.udh_last_error()


def test_fc1_debug_entry_rejects_bad_arguments():
    """udh_debug_fc1 / udh_debug_fc1_scratch_bytes are exported and check their arguments before touching the device."""
    from unsuperviseddeephomographyral2018_b200 import _lib
    L = _lib.lib
    raw = ctypes.CDLL(_lib.LIB_PATH)
    assert hasattr(raw, "udh_debug_fc1") and hasattr(raw, "udh_debug_fc1_scratch_bytes")
    F = 32768
    for B in (1, 129, 512):
        x3, bf = L.udh_debug_fc1_scratch_bytes(B, _lib.NUMERIC_BF16X3), L.udh_debug_fc1_scratch_bytes(B, _lib.NUMERIC_BF16)
        assert x3 >= 4 * (B * F + F * 1024 + B * 1024) and bf >= 2 * (B * F + F * 1024 + B * 1024), B
        assert x3 < 4 * (B * F + F * 1024 + B * 1024) + 1024 and bf < 2 * (B * F + F * 1024 + B * 1024) + 1024, B
    assert L.udh_debug_fc1_scratch_bytes(4, _lib.NUMERIC_FP32) == 0
    assert L.udh_debug_fc1_scratch_bytes(0, _lib.NUMERIC_BF16X3) == 0
    assert L.udh_debug_fc1_scratch_bytes(4, 3) == 0
    p = ctypes.c_void_p(256)                          # never dereferenced: every call below fails its argument checks
    for mode in (_lib.NUMERIC_FP32, _lib.NUMERIC_BF16, _lib.NUMERIC_BF16X3):
        for i in (0, 1, 3, 4, 5, 6):                  # x, w, y; dW and dx when dy is given; scratch in the tensor-core modes
            if i == 6 and mode == _lib.NUMERIC_FP32:
                continue
            a = [p, p, p, p, p, p, p]
            a[i] = None
            assert L.udh_debug_fc1(mode, *a, 4, None) == _lib.EINVAL, (mode, i)
            assert b"udh_debug_fc1: null pointer" in L.udh_last_error()
        assert L.udh_debug_fc1(mode, p, p, p, p, p, p, p, 0, None) == _lib.EINVAL
        assert b"batch must be >= 1" in L.udh_last_error()
        assert L.udh_debug_fc1(mode, p, p, p, p, p, p, p, -3, None) == _lib.EINVAL
    for mode in (-1, 3):
        assert L.udh_debug_fc1(mode, p, p, p, p, p, p, p, 4, None) == _lib.EINVAL
        assert b"unknown numeric_mode" in L.udh_last_error()


def test_fc1_ex_debug_entry_rejects_what_the_step_rejects():
    """udh_debug_fc1_ex (fc1 at any fp32 patch size) checks B and P as udh_cnn_fwd does, and its pointers, before touching
    the device."""
    from unsuperviseddeephomographyral2018_b200 import _lib
    L = _lib.lib
    p = ctypes.c_void_p(256)                          # never dereferenced: every call below fails its argument checks
    for B, P, msg in ((0, 128, b"batch must be >= 1"), (-2, 1408, b"batch must be >= 1"), (1, 100, b"multiple of 128"),
                      (1, 0, b"multiple of 128"), (1, 1536, b"P <= 1408")):
        assert L.udh_debug_fc1_ex(p, p, p, p, p, p, B, P, None) == _lib.EINVAL, (B, P)
        assert msg in L.udh_last_error(), (B, P, L.udh_last_error())
    for i in (0, 1, 3, 4, 5):                         # x, w, y; dW and dx when dy is given
        a = [p, p, p, p, p, p]
        a[i] = None
        assert L.udh_debug_fc1_ex(*a, 2, 1408, None) == _lib.EINVAL, i
        assert b"udh_debug_fc1_ex: null pointer" in L.udh_last_error()


def test_simt_debug_entries_reject_bad_arguments():
    """udh_debug_simt_conv / _wgrad / _pool are exported and check their arguments before touching the device."""
    from unsuperviseddeephomographyral2018_b200 import _lib
    L = _lib.lib
    raw = ctypes.CDLL(_lib.LIB_PATH)
    assert all(hasattr(raw, s) for s in ("udh_debug_simt_conv", "udh_debug_simt_wgrad", "udh_debug_simt_pool"))
    p = ctypes.c_void_p(256)                          # never dereferenced: every call below fails its argument checks
    shape = (2, 16, 16, 64, 64)
    for dgrad, nulls in ((0, (0, 2, 5)), (1, (0, 2, 5, 6))):   # x, w, out; wrot for the dgrad
        for i in nulls:
            a = [p, None, p, None, None, p, p]
            a[i] = None
            assert L.udh_debug_simt_conv(*a, *shape, 0, dgrad, None) == _lib.EINVAL, (dgrad, i)
            assert b"udh_debug_simt_conv: null pointer" in L.udh_last_error()
    conv = lambda x2, bias, B, H, W, cin, cout, relu, dgrad: L.udh_debug_simt_conv(p, x2, p, bias, None, p, p, B, H, W, cin, cout,
                                                                                   relu, dgrad, None)
    assert conv(p, None, 2, 16, 16, 2, 64, 0, 1) == _lib.EINVAL          # dgrad with a second plane
    assert conv(None, p, 2, 16, 16, 64, 64, 0, 1) == _lib.EINVAL         # dgrad with a bias
    assert conv(None, None, 2, 16, 16, 64, 64, 1, 1) == _lib.EINVAL      # dgrad with ReLU
    assert b"the dgrad takes one input" in L.udh_last_error()
    for B, H, W in ((0, 16, 16), (2, 12, 16), (2, 16, 24), (2, 0, 16)):
        assert conv(None, None, B, H, W, 64, 64, 1, 0) == _lib.EINVAL, (B, H, W)
        assert b"needs B >= 1" in L.udh_last_error()
    for x2, cin, cout, dgrad in ((None, 64, 96, 0), (None, 12, 64, 0), (p, 3, 64, 0), (None, 64, 68, 1), (None, 96, 64, 1)):
        assert conv(x2, None, 2, 16, 16, cin, cout, 0, dgrad) == _lib.EINVAL, (cin, cout, dgrad)
        assert b"unsupported channels" in L.udh_last_error()
    part = [ctypes.c_int(-1) for _ in range(3)]
    refs = [ctypes.byref(v) for v in part]
    for i in (0, 2, 3, 4):                            # x, g, dW, db
        a = [p, None, p, p, p]
        a[i] = None
        assert L.udh_debug_simt_wgrad(*a, *shape, *refs, None) == _lib.EINVAL
        assert b"udh_debug_simt_wgrad: null pointer" in L.udh_last_error()
    assert L.udh_debug_simt_wgrad(p, None, p, p, p, 0, 16, 16, 64, 64, *refs, None) == _lib.EINVAL
    assert L.udh_debug_simt_wgrad(p, None, p, p, p, 2, 16, 16, 8, 64, *refs, None) == _lib.EINVAL    # cin % 16
    assert L.udh_debug_simt_wgrad(p, p, p, p, p, 2, 16, 16, 64, 64, *refs, None) == _lib.EINVAL      # two planes need cin == 2
    assert b"unsupported channels" in L.udh_last_error()
    assert [v.value for v in part] == [-1, -1, -1]    # nothing reported for a rejected call
    for a in ((None, p, None, None), (p, None, None, None), (p, None, None, p), (p, None, p, None)):
        assert L.udh_debug_simt_pool(*a, 2, 16, 16, 64, None) == _lib.EINVAL, a
        assert b"udh_debug_simt_pool: null pointer" in L.udh_last_error()
    for B, H, W, C in ((0, 16, 16, 64), (2, 15, 16, 64), (2, 16, 7, 64), (2, 16, 16, 6)):
        assert L.udh_debug_simt_pool(p, p, p, p, B, H, W, C, None) == _lib.EINVAL
        assert b"udh_debug_simt_pool: needs" in L.udh_last_error()


def test_fp32_patch_size_is_limited_by_fc1_weight_gradient_grid():
    """fc1's fp32 weight gradient launches (P/8)^2 * 128 / 64 CTA rows on grid.y (max 65535): P = 1408 is the largest patch
    whose backward can launch, and every entry that takes a patch size rejects a larger one before touching the device."""
    from unsuperviseddeephomographyral2018_b200 import _lib
    L = _lib.lib
    assert (1408 // 8) ** 2 * 128 // 64 <= 65535 < (1536 // 8) ** 2 * 128 // 64
    assert L.udh_cnn_workspace_bytes(1, 1408, _lib.NUMERIC_FP32) > 0
    assert L.udh_cnn_workspace_bytes(1, 256, _lib.NUMERIC_FP32) > 0
    for P in (1536, 2048, 4096):
        assert L.udh_cnn_workspace_bytes(1, P, _lib.NUMERIC_FP32) == 0, P
        assert b"patch size %d is too large" % P in L.udh_last_error()
        assert b"P <= 1408" in L.udh_last_error()
        assert L.udh_cnn_workspace_init(None, 0, 1, P, _lib.NUMERIC_FP32, None) == _lib.EINVAL
        assert b"udh_cnn_workspace_init: patch size %d is too large" % P in L.udh_last_error()
        p = ctypes.c_void_p(256)
        assert L.udh_cnn_fwd(p, p, p, p, p, 1 << 40, 1, P, 0, 0, _lib.NUMERIC_FP32, None) == _lib.EINVAL
        assert L.udh_cnn_bwd(p, p, p, p, p, p, 1 << 40, 1, P, 1, _lib.NUMERIC_FP32, None) == _lib.EINVAL
        assert b"too large" in L.udh_last_error()
    assert L.udh_cnn_workspace_init(None, 0, 1, 1408, _lib.NUMERIC_FP32, None) == _lib.EINVAL
    assert b"bad workspace" in L.udh_last_error()                        # 1408 passes the argument check
    assert L.udh_cnn_workspace_bytes(1, 256, _lib.NUMERIC_BF16X3) == 0   # the tensor-core modes stay at 128
    assert b"tiled for the reference's 128x128 patches" in L.udh_last_error()


def test_schedule_matches_reference_constants():
    from unsuperviseddeephomographyral2018_b200 import engine
    assert engine.decay_steps(1e-4, 0.9e-4) == 58117 and engine.decay_steps(5e-4, 0.9e-4) == 3570
    assert engine.learning_rate(58117, 1e-4, 0.9e-4) == pytest.approx(0.96e-4)
