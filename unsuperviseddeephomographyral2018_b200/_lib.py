"""ctypes binding of libudh.so (include/udh.h).  No CPU fallback: if the library is missing it is built with nvcc,
and if that is impossible the import fails loudly."""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int64, c_size_t, c_uint32, c_uint64, c_ulonglong, c_void_p

from . import build_ext

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = build_ext.lib_path()      # libudh.so (UDH_LIB_VARIANT selects an experimental build variant)

OK, EINVAL, ECUDA, ENOSUP, EWS = 0, -1, -2, -3, -4
NUMERIC_FP32, NUMERIC_BF16, NUMERIC_BF16X3 = 0, 1, 2
BWD_ALL, BWD_HEAD, BWD_CONVS = 0, 1, 2
LOSS_L1, LOSS_REC, LOSS_L1_SMOOTH, LOSS_NCC, LOSS_CUSTOM = 0, 1, 2, 3, 4
NSUMS, NLOSSES, NMETRICS = 8, 8, 4
L_REC, L_SSIM, L_L1, L_L1_SMOOTH, L_NCC = 0, 1, 2, 3, 4
M_H_LOSS, M_BOUNDED_H_LOSS, M_NUM_FAIL, M_ACE = 0, 1, 2, 3
ECC_OK, ECC_NAN, ECC_NOCONV = 0, 1, 2
MOSAIC_TILE_H, MOSAIC_TILE_W = 16, 64            # UDH_MOSAIC_TILE_H / _W
EXPOSURE_MAX_FRAMES, EXPOSURE_MAX_FEEDS, EXPOSURE_STATS = 1024, 16, 13   # UDH_EXPOSURE_MAX_FRAMES / _MAX_FEEDS / _STATS
SEAM_MAX_FRAMES = 1024                            # UDH_SEAM_MAX_FRAMES
EXPOSURE_MAX_BLOCKS = 1 << 24                     # UDH_EXPOSURE_MAX_BLOCKS

class StepArgs(ctypes.Structure):
    """udh_step_args (include/udh.h)."""
    _fields_ = [("B", c_int), ("P", c_int), ("img_h", c_int), ("img_w", c_int), ("C", c_int),
                ("numeric_mode", c_int), ("loss_type", c_int), ("train", c_int), ("seed", c_uint64),
                ("params", c_void_p), ("grads", c_void_p), ("ws", c_void_p), ("ws_bytes", c_size_t),
                ("I1", c_void_p), ("I2", c_void_p), ("I_aug", c_void_p), ("pts1", c_void_p), ("gt", c_void_p),
                ("patch_indices", c_void_p), ("idx_stride", c_int64),
                ("h4p", c_void_p), ("H", c_void_p), ("pred_I2", c_void_p),
                ("dh4p", c_void_p), ("dH", c_void_p), ("scratch", c_void_p), ("dpred_map", c_void_p), ("sums", c_void_p),
                ("photo_losses", c_void_p), ("h4p_metrics", c_void_p), ("per_sample", c_void_p), ("fwd_flags", c_int)]


FWD_FC1_MIRROR_CURRENT = 1


class GainMap(ctypes.Structure):
    """udh_gain_map (include/udh.h): a frame's block gain map and its ROI's resize taps (udh_map_tap: int32 s0, s1,
    float32 a0, a1 per column / row), all device pointers."""
    _fields_ = [("map", c_void_p), ("cols", c_void_p), ("rows", c_void_p), ("bpx", c_int), ("bpy", c_int), ("channels", c_int),
                ("pad", c_int)]


class JpegInfo(ctypes.Structure):
    """udh_jpeg_info (include/udh.h)."""
    _fields_ = [("width", c_int), ("height", c_int), ("components", c_int), ("h_samp", c_int * 3), ("v_samp", c_int * 3),
                ("restart_interval", c_int), ("reason", c_int)]


# udh_jpeg_parse reasons (UDH_JPEG_R_*) and udh_jpeg_decode statuses (UDH_JPEG_E_*)
JPEG_R = dict(OK=0, NOT_JPEG=1, TRUNCATED=2, NOT_BASELINE=3, PRECISION=4, COMPONENTS=5, RGB=6, SAMPLING_H=7, SAMPLING_V=8,
              ORIENTATION=9, MULTI_SCAN=10)
JPEG_E = dict(TRUNCATED=1, HUFFMAN=2, COEF=3)


class PngInfo(ctypes.Structure):
    """udh_png_info (include/udh.h)."""
    _fields_ = [("width", c_int), ("height", c_int), ("bit_depth", c_int), ("color_type", c_int), ("interlace", c_int),
                ("channels", c_int), ("idat_bytes", c_int64), ("reason", c_int), ("pad", c_int)]


# udh_png_parse reasons (UDH_PNG_R_*) and udh_png_decode statuses (UDH_PNG_E_*)
PNG_R = dict(OK=0, NOT_PNG=1, JPEG=2, TRUNCATED=3, IDAT_TRUNCATED=4, CRC=5, NO_IEND=6, MALFORMED=7, PALETTE=8, DEPTH16=9,
             DEPTH_SUB8=10, INTERLACED=11, GRAY_ALPHA=12, CHUNK=13)
PNG_E = dict(TRUNCATED=1, ZLIB=2, BLOCK=3, CODE=4, DISTANCE=5, ADLER=6, SHORT=7, LONG=8, FILTER=9)


STEP_ALL, STEP_FWD_HEAD, STEP_CONVS, STEP_FWD_ONLY = 0, 1, 2, 3
STEP_LOSS = {"h_loss": 0, "l1_loss": 1, "rec_loss": 2, "l1_smooth_loss": 3, "ncc_loss": 4, "ssim_loss": 5}


# name -> (restype, argtypes); every symbol include/udh.h declares
SIGNATURES = {
    "udh_version": (c_int, []),
    "udh_last_error": (c_char_p, []),
    "udh_device_available": (c_int, []),
    "udh_dlt_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "udh_dlt_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "udh_warp_loss_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int,
                                  c_void_p, c_void_p, c_int, c_void_p]),
    "udh_warp_loss_fwd_ex": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int,
                                     c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "udh_warp_loss_bwd": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int,
                                  c_void_p, c_float, c_void_p, c_void_p, c_int, c_void_p]),
    "udh_warp_loss_bwd_ex": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int,
                                     c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_int, c_void_p]),
    "udh_ssim_bwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p]),
    "udh_ssim_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p]),
    "udh_photo_losses_finalize": (c_int, [c_void_p, c_double, c_double, c_void_p, c_void_p]),
    "udh_transformer_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "udh_h4p_loss": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "udh_cnn_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "udh_cnn_workspace_init": (c_int, [c_void_p, c_size_t, c_int, c_int, c_int, c_void_p]),
    "udh_cnn_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_int, c_int, c_uint64, c_int,
                            c_void_p]),
    "udh_cnn_fwd_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_int, c_int, c_uint64, c_int,
                               c_int, c_void_p]),
    "udh_cnn_fc1_mirror": (c_int, [c_void_p, c_size_t, c_int, c_int, c_int, POINTER(c_void_p), POINTER(c_size_t), POINTER(c_size_t),
                                   POINTER(c_int)]),
    "udh_cnn_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_int, c_int, c_int,
                            c_void_p]),
    "udh_cnn_bwd_phase": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_int, c_int, c_int,
                                  c_int, c_void_p]),
    "udh_cnn_dropout_masks": (c_int, [c_void_p, c_size_t, c_int, c_int, c_int, POINTER(c_void_p), POINTER(c_void_p)]),
    "udh_cnn_activation": (c_int, [c_void_p, c_size_t, c_int, c_int, c_int, c_int, POINTER(c_void_p), POINTER(c_size_t)]),
    "udh_param_offset": (c_int, [c_int, c_int, POINTER(c_size_t), POINTER(c_size_t)]),
    "udh_param_total_floats": (c_size_t, [c_int]),
    "udh_adam_step": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_float, c_float, c_float, c_float, c_float,
                              c_int, c_void_p]),
    "udh_adam_step_mirror": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_float, c_float, c_float, c_float, c_float,
                                     c_int, c_void_p, c_size_t, c_size_t, c_int, c_void_p]),
    "udh_adam_step_mirror_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_float, c_float, c_float, c_float, c_float,
                                        c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_void_p]),
    "udh_dp_shard_update": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_size_t, c_size_t, c_size_t,
                                    c_int, c_float, c_float, c_float, c_float, c_float, c_int, c_void_p]),
    "udh_debug_x3_materialize": (c_int, [c_void_p, c_size_t, c_int, c_int, POINTER(c_size_t), c_void_p]),
    "udh_debug_x3_set_rows": (c_int, [c_int]),
    "udh_debug_x3_scratch_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "udh_debug_x3_conv": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                  c_void_p]),
    "udh_debug_x3_conv_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                     c_int, c_int, c_int, c_void_p]),
    "udh_debug_x3_conv_rows": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                       c_void_p]),
    "udh_debug_x3_wgrad": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "udh_debug_x3_conv1": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                   c_int, c_void_p]),
    "udh_debug_x3_conv1_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_int, c_int, c_int, c_void_p]),
    "udh_debug_tc_conv_scratch_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "udh_debug_tc_conv": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                          c_void_p]),
    "udh_debug_tc_conv_pool": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "udh_debug_tc_wgrad": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "udh_debug_tc_pool": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "udh_debug_fc1_scratch_bytes": (c_size_t, [c_int, c_int]),
    "udh_debug_fc1": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "udh_debug_fc1_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "udh_debug_simt_conv": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                    c_int, c_int, c_int, c_void_p]),
    "udh_debug_simt_wgrad": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                     POINTER(c_int), POINTER(c_int), POINTER(c_int), c_void_p]),
    "udh_debug_simt_pool": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "udh_step_forward_backward": (c_int, [POINTER(StepArgs), c_int, c_void_p]),
    "udh_prep_inputs_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                   c_void_p]),
    "udh_prep_inputs_u8_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "udh_synth_scene_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_uint64, c_void_p]),
    "udh_warp_image_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "udh_ecc_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "udh_ecc_prep_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "udh_ecc_homography": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_double, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_size_t, c_int, c_int, c_int, c_void_p]),
    "udh_ecc_split_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "udh_ecc_homography_split": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_double, c_void_p, c_void_p, c_void_p, c_void_p,
                                         c_void_p, c_size_t, c_int, c_int, c_int, c_void_p]),
    "udh_debug_ecc_layout": (c_int, [c_int, c_int, c_int, POINTER(c_size_t), POINTER(c_int)]),
    "udh_ecc_h4p": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "udh_ecc_corr_h4p": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "udh_resize_area_up_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "udh_resize_linear_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "udh_real_prep_smem_bytes": (c_size_t, [c_int, c_int]),
    "udh_real_prep": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                              c_void_p, c_void_p, c_void_p]),
    "udh_jpeg_parse": (c_int, [c_void_p, c_int64, POINTER(JpegInfo)]),
    "udh_jpeg_plan_bytes": (c_size_t, [c_void_p, c_void_p, c_int, c_int, c_int]),
    "udh_jpeg_plan": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_size_t]),
    "udh_jpeg_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "udh_jpeg_decode": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "udh_debug_jpeg_set_lanes": (c_int, [c_int]),
    "udh_jpeg_plan_workspace_bytes": (c_size_t, [c_void_p]),
    "udh_debug_jpeg_set_parallel": (c_int, [c_int]),
    "udh_debug_jpeg_set_sync_rounds": (c_int, [c_int]),
    "udh_debug_jpeg_parallel_segments": (c_int, [c_void_p, c_void_p, POINTER(c_int)]),
    "udh_png_parse": (c_int, [c_void_p, c_int64, POINTER(PngInfo)]),
    "udh_png_plan_bytes": (c_size_t, [c_void_p, c_void_p, c_int, c_int, c_int, POINTER(c_int64)]),
    "udh_png_plan": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p, c_int64]),
    "udh_png_workspace_bytes": (c_size_t, [c_void_p]),
    "udh_png_decode": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_size_t, c_void_p]),
    "udh_jpeg_encode_capacity": (c_int64, [c_int, c_int, c_int]),
    "udh_jpeg_encode_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "udh_jpeg_encode": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int64, c_void_p, c_void_p, c_void_p,
                                c_size_t, c_void_p]),
    "udh_gen_warp_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "udh_gray_u8": (c_int, [c_void_p, c_int64, c_void_p, c_void_p]),
    "udh_warp_perspective_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "udh_mosaic_workspace_bytes": (c_size_t, [c_int]),
    "udh_mosaic_blend_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                    c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "udh_mosaic_multiband_workspace_bytes": (c_size_t, [c_void_p, c_int, c_int, c_int, c_int]),
    "udh_mosaic_multiband_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                        c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "udh_debug_multiband_layout": (c_int, [c_void_p, c_int, c_int, c_int, c_int, POINTER(c_size_t), POINTER(c_int)]),
    "udh_mosaic_exposure_workspace_bytes": (c_size_t, [c_int]),
    "udh_mosaic_exposure_stats_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int,
                                             c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "udh_mosaic_seam_workspace_bytes": (c_size_t, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int]),
    "udh_mosaic_seam_masks_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                         c_void_p, c_void_p, c_size_t, c_void_p]),
    "udh_mosaic_seam_gc_workspace_bytes": (c_size_t, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int]),
    "udh_mosaic_seam_gc_masks_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                            c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "udh_debug_grid_mincut_workspace_bytes": (c_size_t, [c_int, c_int]),
    "udh_debug_grid_mincut": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_size_t, c_void_p]),
    "udh_resize_linear_exact_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "udh_mosaic_seam_upscale_workspace_bytes": (c_size_t, [c_void_p, c_void_p, c_int, c_int, c_int, c_double, c_int, c_int]),
    "udh_mosaic_seam_upscale_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_double,
                                           c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "udh_mosaic_exposure_block_workspace_bytes": (c_size_t, [c_int]),
    "udh_mosaic_exposure_block_stats_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int64, c_void_p,
                                                   c_void_p, c_int, c_void_p, c_void_p, c_int64, c_void_p, c_int, c_int, c_int, c_int,
                                                   c_void_p, c_void_p, c_size_t, c_void_p]),
    "udh_exposure_block_solve_workspace_bytes": (c_size_t, [c_int]),
    "udh_exposure_block_solve": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_double, c_int, c_void_p, c_void_p, c_void_p,
                                         c_size_t, c_void_p]),
    "udh_exposure_gain_maps_workspace_bytes": (c_size_t, [c_int64, c_int]),
    "udh_exposure_gain_maps": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "udh_draw_report_workspace_bytes": (c_size_t, [c_int]),
    "udh_draw_report_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_int, c_int,
                                   c_void_p]),
    "udh_launch_count": (c_ulonglong, []),
    "udh_set_sm_reserve": (c_int, [c_int]),
    "udh_set_sm_reserve_top": (c_int, [c_int]),
    "udh_set_adam_grid": (c_int, [c_int]),
    "udh_crc32c": (c_uint32, [c_void_p, c_size_t, c_uint32]),
    "udh_set_bwd_marker": (c_int, [c_int]),
    "udh_set_sm_reserve_marker": (c_int, [c_int]),
    "udh_bwd_marker_wait": (c_int, [c_void_p]),
    "udh_prof_enable": (c_int, [c_int]),
    "udh_prof_reset": (c_int, []),
    "udh_prof_num_tags": (c_int, []),
    "udh_prof_tag_name": (c_char_p, [c_int]),
    "udh_prof_read": (c_int, [c_int, POINTER(c_float), POINTER(c_int)]),
}


class UdhError(RuntimeError):
    pass


def _load():
    if build_ext.needs_build():
        build_ext.build()      # raises if nvcc is unavailable: there is deliberately no pure-Python/CPU path
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


def check(rc, what=""):
    if rc != OK:
        raise UdhError("%s failed (%d): %s" % (what or "libudh call", rc, lib.udh_last_error().decode()))


def require_device():
    if not lib.udh_device_available():
        raise UdhError("no CUDA device: libudh has no CPU fallback (the CPU oracle lives in oracle/ and is test-only)")


def prof_read_all():
    """{tag name: (total_ms, count)} of the library's per-phase CUDA-event timers (non-empty phases only)."""
    out = {}
    for t in range(lib.udh_prof_num_tags()):
        ms, n = c_float(), c_int()
        check(lib.udh_prof_read(t, ctypes.byref(ms), ctypes.byref(n)), "udh_prof_read")
        if n.value:
            out[lib.udh_prof_tag_name(t).decode()] = (ms.value, n.value)
    return out
