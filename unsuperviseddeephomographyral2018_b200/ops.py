"""Torch-tensor wrappers over the C ABI (include/udh.h).  PyTorch is plumbing here: device memory, streams and
autograd bookkeeping; all arithmetic happens in libudh's CUDA kernels.  Every function requires CUDA tensors."""
import ctypes
import functools
import math

import numpy as np
import torch

from . import _lib
from ._lib import check, lib


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _req(t, dtype, name):
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise _lib.UdhError("%s must be a CUDA tensor (libudh has no CPU path)" % name)
    if t.dtype != dtype or not t.is_contiguous():
        raise _lib.UdhError("%s must be contiguous %s (got %s, contiguous=%s)" % (name, dtype, t.dtype, t.is_contiguous()))
    return t


# ------------------------------------------------------------------ Row D: DLT
def dlt_forward(pts1, h4p):
    """pts1, h4p [B,8] -> H [B,3,3] (reference HomographyModel.solve_DLT, homography_model.py:169-250)."""
    _req(pts1, torch.float32, "pts1"); _req(h4p, torch.float32, "h4p")
    B = pts1.shape[0]
    H = torch.empty(B, 3, 3, device=pts1.device, dtype=torch.float32)
    check(lib.udh_dlt_fwd(_ptr(pts1), _ptr(h4p), _ptr(H), B, _stream()), "udh_dlt_fwd")
    return H


def dlt_backward(pts1, h4p, H, dH):
    _req(dH, torch.float32, "dH")
    B = pts1.shape[0]
    dh4p = torch.empty(B, 8, device=pts1.device, dtype=torch.float32)
    check(lib.udh_dlt_bwd(_ptr(pts1), _ptr(h4p), _ptr(H), _ptr(dH), _ptr(dh4p), B, _stream()), "udh_dlt_bwd")
    return dh4p


class SolveDLT(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pts1, h4p):
        pts1 = pts1.contiguous(); h4p = h4p.contiguous()
        H = dlt_forward(pts1, h4p)
        ctx.save_for_backward(pts1, h4p, H)
        return H

    @staticmethod
    def backward(ctx, dH):
        pts1, h4p, H = ctx.saved_tensors
        return None, dlt_backward(pts1, h4p, H, dH.contiguous())


solve_dlt = SolveDLT.apply


# ------------------------------------------------------------------ Rows W + L: fused warp + photometric losses
def _img_args(I):
    B, Hh, W, C = I.shape
    return B, Hh, W, C


def warp_loss_forward(I, H, I2, patch_indices, pw, ph, want_pred=True, sums=None):
    """I [B,Hh,W,C], H [B,3,3] pixel units, I2 [B,ph,pw(,1)] or None, patch_indices [B,ph*pw] int32 or None.
    Returns (pred_I2 [B,ph,pw,1] or None, sums double[8])."""
    _req(I, torch.float32, "I"); _req(H, torch.float32, "H")
    B, Hh, W, C = _img_args(I)
    if I2 is not None:
        _req(I2, torch.float32, "I2")
    stride = 0
    if patch_indices is not None:
        _req(patch_indices, torch.int32, "patch_indices")
        stride = patch_indices.stride(0) if patch_indices.dim() > 1 else 1
    pred = torch.empty(B, ph, pw, 1, device=I.device, dtype=torch.float32) if want_pred else None
    if sums is None:
        sums = torch.zeros(_lib.NSUMS, device=I.device, dtype=torch.float64)
    check(lib.udh_warp_loss_fwd(_ptr(I), C, Hh, W, _ptr(H), _ptr(I2), _ptr(patch_indices), stride, pw, ph, _ptr(pred),
                                _ptr(sums), B, _stream()), "udh_warp_loss_fwd")
    return pred, sums


def ssim_backward(pred, I2, pw, ph):
    """d ssim_loss / d pred [B,ph,pw] (homography_model.py:141-158,316)."""
    B = pred.shape[0]
    dpred = torch.empty(B, ph, pw, device=pred.device, dtype=torch.float32)
    check(lib.udh_ssim_bwd(_ptr(pred), _ptr(I2), pw, ph, _ptr(dpred), B, _stream()), "udh_ssim_bwd")
    return dpred


def warp_loss_backward(I, H, I2, patch_indices, pw, ph, loss_type, sums, upstream=1.0, dpred=None):
    B, Hh, W, C = _img_args(I)
    stride = 0
    if patch_indices is not None:
        stride = patch_indices.stride(0) if patch_indices.dim() > 1 else 1
    dH = torch.empty(B, 3, 3, device=I.device, dtype=torch.float32)
    scratch = torch.empty(B * 9, device=I.device, dtype=torch.float32)
    check(lib.udh_warp_loss_bwd_ex(_ptr(I), C, Hh, W, _ptr(H), _ptr(I2), _ptr(patch_indices), stride, pw, ph, loss_type,
                                   _ptr(sums), _ptr(dpred), float(upstream), _ptr(dH), _ptr(scratch), B, _stream()), "udh_warp_loss_bwd_ex")
    return dH


def photo_losses(pred, I2, sums, pw, ph, B):
    """SSIM pass + finalisation -> float tensor [8] indexed by _lib.L_* (rec, ssim, l1, l1_smooth, ncc)."""
    check(lib.udh_ssim_fwd(_ptr(pred), _ptr(I2), pw, ph, _ptr(sums), B, _stream()), "udh_ssim_fwd")
    out = torch.empty(_lib.NLOSSES, device=pred.device, dtype=torch.float32)
    check(lib.udh_photo_losses_finalize(_ptr(sums), float(B * pw * ph), float(B * (pw - 2) * (ph - 2)), _ptr(out), _stream()),
          "udh_photo_losses_finalize")
    return out


_LOSS_SLOT = {_lib.LOSS_L1: _lib.L_L1, _lib.LOSS_REC: _lib.L_REC, _lib.LOSS_L1_SMOOTH: _lib.L_L1_SMOOTH}


class WarpPhotoLoss(torch.autograd.Function):
    """loss(H) for loss_type in {L1, REC, L1_SMOOTH}; differentiable w.r.t. H only (the image is data)."""

    @staticmethod
    def forward(ctx, H, I, I2, patch_indices, pw, ph, loss_type):
        H = H.contiguous()
        pred, sums = warp_loss_forward(I, H, I2, patch_indices, pw, ph, want_pred=False)
        out = torch.empty(_lib.NLOSSES, device=I.device, dtype=torch.float32)
        B = I.shape[0]
        check(lib.udh_photo_losses_finalize(_ptr(sums), float(B * pw * ph), 0.0, _ptr(out), _stream()), "finalize")
        ctx.save_for_backward(H, I, I2, patch_indices, sums)
        ctx.cfg = (pw, ph, loss_type)
        return out[_LOSS_SLOT[loss_type]].clone()

    @staticmethod
    def backward(ctx, gout):
        H, I, I2, patch_indices, sums = ctx.saved_tensors
        pw, ph, loss_type = ctx.cfg
        dH = warp_loss_backward(I, H, I2, patch_indices, pw, ph, loss_type, sums, 1.0)
        return dH * gout, None, None, None, None, None, None


def warp_photo_loss(H, I, I2, patch_indices, pw, ph, loss_type=_lib.LOSS_L1):
    return WarpPhotoLoss.apply(H, I, I2, patch_indices, pw, ph, loss_type)


# ------------------------------------------------------------------ the `transformer` operator
def transformer(U, theta, out_size, name="SpatialTransformer", **kwargs):
    """Drop-in for utils/tf_spatial_transformer.py:18 `transformer(U, theta, out_size)`:
    U [B,H,W,C] float32, theta [B,3,3] or [B,9] normalised homography, out_size (out_h, out_w).
    Returns (output [B,out_h,out_w,C], condition) — `condition` (tf_spatial_transformer.py:235, the count of
    |t_s| > 1e-7 which no caller reads) is returned as None."""
    _req(U, torch.float32, "U")
    theta = theta.reshape(-1, 9).contiguous()
    _req(theta, torch.float32, "theta")
    B, H, W, C = U.shape
    oh, ow = int(out_size[0]), int(out_size[1])
    out = torch.empty(B, oh, ow, C, device=U.device, dtype=torch.float32)
    check(lib.udh_transformer_fwd(_ptr(U), _ptr(theta), _ptr(out), B, H, W, C, oh, ow, _stream()), "udh_transformer_fwd")
    return out, None


# ------------------------------------------------------------------ h4p losses / metrics
def h4p_loss(pred, gt, want_grad=False, want_per_sample=False):
    """-> (metrics float[4] indexed by _lib.M_*, per_sample [B] or None, dpred [B,8] or None)."""
    _req(pred, torch.float32, "pred_h4p"); _req(gt, torch.float32, "gt")
    B = pred.shape[0]
    metrics = torch.empty(_lib.NMETRICS, device=pred.device, dtype=torch.float32)
    per = torch.empty(B, device=pred.device, dtype=torch.float32) if want_per_sample else None
    dpred = torch.empty(B, 8, device=pred.device, dtype=torch.float32) if want_grad else None
    check(lib.udh_h4p_loss(_ptr(pred), _ptr(gt), B, _ptr(metrics), _ptr(per), _ptr(dpred), _stream()), "udh_h4p_loss")
    return metrics, per, dpred


# ------------------------------------------------------------------ direct method (cv2.findTransformECC, MOTION_HOMOGRAPHY)
def ecc_prep_u8(I_u8, Ip_u8, aug=None):
    """Decoded I, I' [B,H,W,3] uint8 (+ the [B,11] augmentation table or None) -> the two uint8 gray planes [B,H,W] the
    reference hands to ECC: cvtColor(denorm_img(I_aug).astype(uint8), RGB2GRAY)."""
    _req(I_u8, torch.uint8, "I"); _req(Ip_u8, torch.uint8, "I_prime")
    if aug is not None:
        _req(aug, torch.float32, "aug")
    B, Hh, W, _ = I_u8.shape
    g1 = torch.empty(B, Hh, W, device=I_u8.device, dtype=torch.uint8)
    g2 = torch.empty_like(g1)
    check(lib.udh_ecc_prep_u8(_ptr(I_u8), _ptr(Ip_u8), _ptr(aug), _ptr(g1), _ptr(g2), B, Hh, W, _stream()), "udh_ecc_prep_u8")
    return g1, g2


def find_homography_ecc(template, image, W_init=None, max_iters=8, eps=1e-10):
    """Batched cv2.findTransformECC(template, image, W, MOTION_HOMOGRAPHY, (COUNT|EPS, max_iters, eps)) on uint8 planes
    [B,H,W].  Returns (W [B,3,3] fp32, rho [B] fp64, iterations [B] int32, status [B] int32 in _lib.ECC_*)."""
    return _ecc_call("udh_ecc_homography", "udh_ecc_workspace_bytes", template, image, W_init, max_iters, eps)


def find_homography_ecc_split(template, image, W_init=None, max_iters=8, eps=1e-10):
    """find_homography_ecc with each pair's pixel sums split over many CTAs (udh_ecc_homography_split): for a few large
    pairs.  Same arguments and outputs; a pair's result does not depend on the rest of the batch."""
    return _ecc_call("udh_ecc_homography_split", "udh_ecc_split_workspace_bytes", template, image, W_init, max_iters, eps)


def _ecc_call(fn, ws_fn, template, image, W_init, max_iters, eps):
    _req(template, torch.uint8, "template"); _req(image, torch.uint8, "image")
    if template.shape != image.shape or template.dim() != 3:
        raise _lib.UdhError("template and image must both be [B,H,W] (got %s and %s)" % (tuple(template.shape), tuple(image.shape)))
    B, Hh, W = template.shape
    if W_init is not None:
        W_init = W_init.reshape(B, 9).contiguous()
        _req(W_init, torch.float32, "W_init")
    dev = template.device
    Wout = torch.empty(B, 3, 3, device=dev, dtype=torch.float32)
    rho = torch.empty(B, device=dev, dtype=torch.float64)
    iters = torch.empty(B, device=dev, dtype=torch.int32)
    status = torch.empty(B, device=dev, dtype=torch.int32)
    nbytes = getattr(lib, ws_fn)(B, Hh, W)
    ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    check(getattr(lib, fn)(_ptr(template), _ptr(image), _ptr(W_init), int(max_iters), float(eps), _ptr(Wout), _ptr(rho),
                           _ptr(iters), _ptr(status), _ptr(ws), nbytes, B, Hh, W, _stream()), fn)
    return Wout, rho, iters, status


def ecc_h4p(W, status, pts1, gt=None, rho=45.0):
    """-> (pred_h4p [B,8], h_loss [B] or None, fail [B] int32 or None): the direct method's corner displacements and the
    harness's clamp / failure rules (0 = ok, 1 = not found, 2 = worse than identity)."""
    W = W.reshape(-1, 9).contiguous()
    _req(W, torch.float32, "W"); _req(status, torch.int32, "status"); _req(pts1, torch.float32, "pts1")
    if gt is not None:
        _req(gt, torch.float32, "gt")
    B = W.shape[0]
    pred = torch.empty(B, 8, device=W.device, dtype=torch.float32)
    h = torch.empty(B, device=W.device, dtype=torch.float32) if gt is not None else None
    fail = torch.empty(B, device=W.device, dtype=torch.int32) if gt is not None else None
    check(lib.udh_ecc_h4p(_ptr(W), _ptr(status), _ptr(pts1), _ptr(gt), float(rho), _ptr(pred), _ptr(h), _ptr(fail), B, _stream()),
          "udh_ecc_h4p")
    return pred, h, fail


def ecc_corr_h4p(W, status, gt):
    """The real-data harness's metric on clicked correspondences gt [B,16] (480x640 frame): -> (pred_h4p [B,8] fp32,
    h_loss [B] float64, fail [B] int32: 0 ok, 1 not found, 2 worse than identity).  W is not inverted; see include/udh.h."""
    W = W.reshape(-1, 9).contiguous()
    _req(W, torch.float32, "W"); _req(status, torch.int32, "status"); _req(gt, torch.float32, "gt")
    B = W.shape[0]
    pred = torch.empty(B, 8, device=W.device, dtype=torch.float32)
    h = torch.empty(B, device=W.device, dtype=torch.float64)
    fail = torch.empty(B, device=W.device, dtype=torch.int32)
    check(lib.udh_ecc_corr_h4p(_ptr(W), _ptr(status), _ptr(gt), _ptr(pred), _ptr(h), _ptr(fail), B, _stream()), "udh_ecc_corr_h4p")
    return pred, h, fail


# ------------------------------------------------------------------ real-data input pipeline (cv2.resize INTER_AREA)
def area_is_generic(src_h, src_w, dst_h, dst_w):
    """True when cv2.resize(INTER_AREA) downscales with its generic resizeArea (the path udh_real_prep restates): scale
    >= 1 on both axes, and not an integer ratio on both (that takes resizeAreaFast, another summation order)."""
    if dst_h > src_h or dst_w > src_w:
        return False
    eps = np.finfo(np.float64).eps
    sx, sy = src_w / dst_w, src_h / dst_h
    return not (abs(sx - round(sx)) < eps and abs(sy - round(sy)) < eps)


def _area_entries(ssize, dsize):
    """OpenCV's computeResizeAreaTab (imgproc/src/resize.cpp): (offsets [dsize+1], source index, fp32 weight) in table order."""
    scale = 1.0 / (float(dsize) / float(ssize))
    ofs, src, wt = [0], [], []
    for d in range(dsize):
        f1 = d * scale
        f2 = f1 + scale
        cell = min(scale, ssize - f1)
        s1, s2 = int(np.ceil(f1)), int(np.floor(f2))
        s2 = min(s2, ssize - 1)
        s1 = min(s1, s2)
        if s1 - f1 > 1e-3:
            src.append(s1 - 1); wt.append((s1 - f1) / cell)
        for s in range(s1, s2):
            src.append(s); wt.append(1.0 / cell)
        if f2 - s2 > 1e-3:
            src.append(s2); wt.append(min(min(f2 - s2, 1.0), cell) / cell)
        ofs.append(len(src))
    return np.array(ofs, np.int32), np.array(src, np.int32), np.array(wt, np.float32)


@functools.lru_cache(maxsize=8)
def area_table(src_h, src_w, dst_h, dst_w):
    """udh_real_prep's packed area table (int32) and its max_rows, for the generic resizeArea downscale."""
    if not area_is_generic(src_h, src_w, dst_h, dst_w):
        raise _lib.UdhError("INTER_AREA %dx%d -> %dx%d is not the generic resizeArea downscale" % (src_h, src_w, dst_h, dst_w))
    xo, xs, xw = _area_entries(src_w, dst_w)
    yo, ys, yw = _area_entries(src_h, dst_h)
    tab = np.concatenate([[len(xs), len(ys)], xo, xs, xw.view(np.int32), yo, ys, yw.view(np.int32)]).astype(np.int32)
    return tab, int(np.diff(yo).max())


@functools.lru_cache(maxsize=8)
def linear_area_table(src_h, src_w, dst_h, dst_w):
    """udh_resize_area_up_u8's table (int32): INTER_AREA upscaling is linear interpolation with area coefficients —
    fx = (d+1) - (s+1) inv_scale in float, fx - floor(fx), 11-bit fixed point (cvRound), both taps on the last pixel at
    the right / bottom border."""
    def axis(ssize, dsize):
        inv = float(dsize) / float(ssize)
        s_, a0, a1 = [], [], []
        for d in range(dsize):
            s = int(np.floor(d * (1.0 / inv)))
            fx = np.float32((d + 1) - (s + 1) * inv)
            fx = np.float32(0) if fx <= 0 else np.float32(fx - np.floor(fx))
            c0, c1 = np.float32(1) - fx, fx
            if s >= ssize - 1:
                s, c0, c1 = ssize - 1, np.float32(1), np.float32(0)
            s_.append(s); a0.append(np.rint(c0 * np.float32(2048))); a1.append(np.rint(c1 * np.float32(2048)))
        return [s_, a0, a1]
    if not (dst_h > src_h and dst_w > src_w):
        raise _lib.UdhError("udh_resize_area_up_u8 upscales on both axes (got %dx%d -> %dx%d)" % (src_h, src_w, dst_h, dst_w))
    return np.concatenate([np.array(a, np.float64) for a in axis(src_w, dst_w) + axis(src_h, dst_h)]).astype(np.int32)


def resize_area_up_u8(src, dst_h, dst_w):
    """uint8 [N,h,w,3] CUDA tensor -> [N,dst_h,dst_w,3]: cv2.resize(INTER_AREA) per image, bit for bit."""
    _req(src, torch.uint8, "src")
    n, h, w, _ = src.shape
    tab = torch.from_numpy(linear_area_table(h, w, dst_h, dst_w)).to(src.device)
    out = torch.empty(n, dst_h, dst_w, 3, device=src.device, dtype=torch.uint8)
    check(lib.udh_resize_area_up_u8(_ptr(src), _ptr(tab), _ptr(out), n, h, w, dst_h, dst_w, _stream()), "udh_resize_area_up_u8")
    return out


@functools.lru_cache(maxsize=32)
def linear_table(src_h, src_w, dst_h, dst_w):
    """udh_resize_linear_u8's table (int32): xsrc, xa0, xa1, ysrc, ya0, ya1, ysrc1 — OpenCV's INTER_LINEAR tables:
    f = (float)((d + 0.5) * scale - 0.5), s = floor(f), f -= s in float, coefficients cvRound((1 - f) * 2048) and
    cvRound(f * 2048) in float.  Columns: s < 0 takes (0, f = 0) and s >= size - 1 takes (size - 1, f = 0).  Rows keep
    their coefficients; the two source rows s and s + 1 are clamped to the image instead."""
    def axis(ssize, dsize, rows):
        scale = 1.0 / (float(dsize) / float(ssize))
        f = ((np.arange(dsize, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
        s = np.floor(f).astype(np.int64)
        f = (f - s.astype(np.float32)).astype(np.float32)
        if rows:
            s0, s1 = np.clip(s, 0, ssize - 1), np.clip(s + 1, 0, ssize - 1)
        else:
            lo, hi = s < 0, s >= ssize - 1
            f[lo | hi] = 0
            s0 = np.clip(s, 0, ssize - 1)
        out = [s0, np.rint((np.float32(1) - f) * np.float32(2048)), np.rint(f * np.float32(2048))]
        return out + [s1] if rows else out
    if min(src_h, src_w, dst_h, dst_w) < 1:
        raise _lib.UdhError("linear_table: sizes must be >= 1 (got %dx%d -> %dx%d)" % (src_h, src_w, dst_h, dst_w))
    return np.concatenate([np.asarray(a, np.float64) for a in axis(src_w, dst_w, False) + axis(src_h, dst_h, True)]).astype(np.int32)


def resize_linear_u8(src, dst_h, dst_w):
    """uint8 [N,h,w,3] CUDA tensor -> [N,dst_h,dst_w,3]: cv2.resize(img, (dst_w, dst_h)) (INTER_LINEAR) per image, bit
    for bit, downscales and upscales.  One launch per source size."""
    _req(src, torch.uint8, "src")
    if src.dim() != 4 or src.shape[3] != 3:
        raise _lib.UdhError("resize_linear_u8: src must be [N,h,w,3] (got %s)" % (tuple(src.shape),))
    n, h, w, _ = src.shape
    tab = torch.from_numpy(linear_table(h, w, dst_h, dst_w)).to(src.device)
    out = torch.empty(n, dst_h, dst_w, 3, device=src.device, dtype=torch.uint8)
    check(lib.udh_resize_linear_u8(_ptr(src), _ptr(tab), _ptr(out), n, h, w, dst_h, dst_w, _stream()), "udh_resize_linear_u8")
    return out


def linear_exact_table(src_h, src_w, dst_h, dst_w, scale=None):
    """udh_resize_linear_exact_u8's table (int32): xs0, xs1, xc1, ys0, ys1, yc1 - cv2's INTER_LINEAR_EXACT taps (the rule:
    oracle/seam_scale.py): per axis the sampling scale is 1 / scale (cv2.resize's fx / fy form) or src / dst (its dsize
    form), f = (d + 0.5) * that - 0.5 in float64, s = floor(f), c1 = rint((f - s) * 256) (ties to even), taps (s, s + 1),
    both on pixel 0 when s < 0 and on pixel size - 1 when s + 1 > size - 1.  An output of the source's size is a copy (cv2's
    rule), the identity table."""
    def axis(n, N, inv):
        f = (np.arange(N, dtype=np.float64) + 0.5) * (1.0 / inv) - 0.5
        s = np.floor(f)
        c1 = np.rint((f - s) * 256.0)
        s = s.astype(np.int64)
        lo, hi = s < 0, s + 1 > n - 1
        return [np.where(lo, 0, np.where(hi, n - 1, s)), np.where(lo, 0, np.where(hi, n - 1, s + 1)), c1]
    if min(src_h, src_w, dst_h, dst_w) < 1:
        raise _lib.UdhError("linear_exact_table: sizes must be >= 1 (got %dx%d -> %dx%d)" % (src_h, src_w, dst_h, dst_w))
    ix = float(scale) if scale is not None else dst_w / float(src_w)
    iy = float(scale) if scale is not None else dst_h / float(src_h)
    if (dst_h, dst_w) == (src_h, src_w):                            # cv2 copies when the size stays, whatever fx says
        ix = iy = 1.0
    return np.concatenate([np.asarray(a, np.float64) for a in axis(src_w, dst_w, ix) + axis(src_h, dst_h, iy)]).astype(np.int32)


def resize_linear_exact_u8(src, dst_h=None, dst_w=None, scale=None):
    """uint8 [N,h,w,C] or [h,w,C] CUDA tensor (C = 1 or 3) -> [N,dst_h,dst_w,C] (or [dst_h,dst_w,C]): cv2.resize with
    INTER_LINEAR_EXACT per image, byte for byte.  Give dst_h and dst_w (cv2.resize(img, (dst_w, dst_h), ...)) or scale
    (cv2.resize(img, None, fx=scale, fy=scale, ...): the sides are rint(side * scale) and the sampling scale is 1 / scale,
    which differs from the dsize form's side / dst).  One launch."""
    _req(src, torch.uint8, "src")
    batched = src.dim() == 4
    if src.dim() not in (3, 4) or src.shape[-1] not in (1, 3):
        raise _lib.UdhError("resize_linear_exact_u8: src must be [N,h,w,C] or [h,w,C] with C = 1 or 3 (got %s)" % (tuple(src.shape),))
    x = src if batched else src[None]
    n, h, w, C = (int(v) for v in x.shape)
    if (scale is None) == (dst_h is None or dst_w is None) or (scale is not None and (dst_h is not None or dst_w is not None)):
        raise _lib.UdhError("resize_linear_exact_u8: give dst_h and dst_w, or scale")
    if scale is not None:
        if not float(scale) > 0:
            raise _lib.UdhError("resize_linear_exact_u8: scale must be > 0 (got %r)" % (scale,))
        dst_h, dst_w = int(np.rint(h * float(scale))), int(np.rint(w * float(scale)))
    tab = torch.from_numpy(linear_exact_table(h, w, int(dst_h), int(dst_w), scale)).to(src.device)
    out = torch.empty(n, int(dst_h), int(dst_w), C, device=src.device, dtype=torch.uint8)
    check(lib.udh_resize_linear_exact_u8(_ptr(x), _ptr(tab), _ptr(out), n, h, w, C, int(dst_h), int(dst_w), _stream()),
          "udh_resize_linear_exact_u8")
    return out if batched else out[0]


def real_prep(I_u8, Ip_u8, luts, img_h, img_w):
    """Full-size uint8 I, I' [B,FH,FW,3] and per-sample value tables luts [B,4,256,3] fp32 (plain I, plain I', augmented I,
    augmented I') -> (I, I_prime, I_aug, I_prime_aug) [B,img_h,img_w,3] fp32: table lookup, then cv2's INTER_AREA
    downscale when the sizes differ — the real-data loader's host arithmetic, bit for bit."""
    _req(I_u8, torch.uint8, "I"); _req(Ip_u8, torch.uint8, "I_prime"); _req(luts, torch.float32, "luts")
    B, FH, FW, _ = I_u8.shape
    tab, max_rows = None, 0
    if (FH, FW) != (img_h, img_w):
        t, max_rows = area_table(FH, FW, img_h, img_w)
        tab = torch.from_numpy(t).to(I_u8.device, non_blocking=True)
    outs = [torch.empty(B, img_h, img_w, 3, device=I_u8.device, dtype=torch.float32) for _ in range(4)]
    check(lib.udh_real_prep(_ptr(I_u8), _ptr(Ip_u8), _ptr(luts), _ptr(tab), max_rows, B, FH, FW, img_h, img_w, *[_ptr(o) for o in outs],
                            _stream()), "udh_real_prep")
    return outs


# ------------------------------------------------------------------ baseline-JPEG decode
def jpeg_parse(blob):
    """One file's bytes -> _lib.JpegInfo (host only): size, sampling, restart interval and `reason`, 0 when the device
    decoder takes the file, else one of _lib.JPEG_R."""
    info = _lib.JpegInfo()
    buf = np.frombuffer(blob, np.uint8) if len(blob) else np.zeros(1, np.uint8)
    check(lib.udh_jpeg_parse(buf.ctypes.data, len(blob), ctypes.byref(info)), "udh_jpeg_parse")
    return info


class JpegPlan:
    """Host side of one decode launch: the files concatenated in pinned memory and the packed descriptor."""

    def __init__(self, blobs, h, w):
        offs = np.zeros(len(blobs) + 1, np.int64)
        offs[1:] = np.cumsum([len(b) for b in blobs])
        self.n, self.h, self.w = len(blobs), h, w
        pin = torch.cuda.is_available()                  # the plan itself is host-only; pinning needs a device
        self.data = torch.empty(max(int(offs[-1]), 1), dtype=torch.uint8, pin_memory=pin)
        dv = self.data.numpy()
        for k, b in enumerate(blobs):
            dv[offs[k]:offs[k + 1]] = np.frombuffer(b, np.uint8)
        nb = lib.udh_jpeg_plan_bytes(dv.ctypes.data, offs.ctypes.data, self.n, h, w)
        if nb == 0:
            raise _lib.UdhError("udh_jpeg_plan_bytes: %s" % lib.udh_last_error().decode())
        self.plan = torch.empty(nb, dtype=torch.uint8, pin_memory=pin)
        check(lib.udh_jpeg_plan(dv.ctypes.data, offs.ctypes.data, self.n, h, w, self.plan.data_ptr(), nb), "udh_jpeg_plan")

    def decode(self, device=None):
        """-> (uint8 [N,h,w,3] RGB, int32 [N] status) on the current stream; nonzero status = that image failed."""
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        plan_d = self.plan.to(dev, non_blocking=True)
        data_d = self.data.to(dev, non_blocking=True)
        out = torch.empty(self.n, self.h, self.w, 3, device=dev, dtype=torch.uint8)
        status = torch.empty(self.n, device=dev, dtype=torch.int32)
        nbytes = lib.udh_jpeg_plan_workspace_bytes(self.plan.data_ptr())
        ws = self.ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)     # kept for udh_debug_jpeg_parallel_segments
        check(lib.udh_jpeg_decode(self.plan.data_ptr(), _ptr(plan_d), _ptr(data_d), _ptr(out), _ptr(status), _ptr(ws), nbytes,
                                  _stream()), "udh_jpeg_decode")
        return out, status


def decode_jpeg(blobs, h, w):
    """Baseline JPEG files (bytes), all h x w -> (uint8 [N,h,w,3] CUDA tensor, int32 [N] status): bit-identical to
    cv2.imread(..., IMREAD_COLOR)[..., ::-1].  Raises UdhError naming the first file the device could not decode."""
    _lib.require_device()
    out, status = JpegPlan(blobs, h, w).decode()
    st = status.cpu().numpy()
    bad = np.flatnonzero(st)
    if len(bad):
        raise _lib.UdhError("decode_jpeg: image %d failed with status %d (%d of %d images failed)" % (bad[0], st[bad[0]], len(bad), len(st)))
    return out, status


# ------------------------------------------------------------------ PNG decode
def png_parse(blob):
    """One file's bytes -> _lib.PngInfo (host only): size, bit depth, colour type, interlace, the zlib stream's length
    and `reason`, 0 when the device decoder takes the file, else one of _lib.PNG_R."""
    info = _lib.PngInfo()
    buf = np.frombuffer(blob, np.uint8) if len(blob) else np.zeros(1, np.uint8)
    check(lib.udh_png_parse(buf.ctypes.data, len(blob), ctypes.byref(info)), "udh_png_parse")
    return info


class PngPlan:
    """Host side of one PNG decode launch: the files' IDAT payloads concatenated in pinned memory (each file's zlib stream
    contiguous) and the per-file descriptor."""

    def __init__(self, blobs, h, w):
        offs = np.zeros(len(blobs) + 1, np.int64)
        offs[1:] = np.cumsum([len(b) for b in blobs])
        self.n, self.h, self.w = len(blobs), h, w
        pin = torch.cuda.is_available()                  # the plan itself is host-only; pinning needs a device
        files = np.zeros(max(int(offs[-1]), 1), np.uint8)
        for k, b in enumerate(blobs):
            files[offs[k]:offs[k + 1]] = np.frombuffer(b, np.uint8)
        nidat = ctypes.c_int64(0)
        nb = lib.udh_png_plan_bytes(files.ctypes.data, offs.ctypes.data, self.n, h, w, ctypes.byref(nidat))
        if nb == 0:
            raise _lib.UdhError("udh_png_plan_bytes: %s" % lib.udh_last_error().decode())
        self.idat = torch.empty(max(nidat.value, 1), dtype=torch.uint8, pin_memory=pin)
        self.plan = torch.empty(nb, dtype=torch.uint8, pin_memory=pin)
        check(lib.udh_png_plan(files.ctypes.data, offs.ctypes.data, self.n, h, w, self.plan.data_ptr(), nb, self.idat.data_ptr(),
                               self.idat.numel()), "udh_png_plan")

    def decode(self, device=None, rgb=False):
        """-> (uint8 [N,h,w,3], int32 [N] status) on the current stream: BGR as cv2.imread returns it (RGB when rgb);
        nonzero status = that image failed (one of _lib.PNG_E) and its output is undefined."""
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        plan_d = self.plan.to(dev, non_blocking=True)
        idat_d = self.idat.to(dev, non_blocking=True)
        out = torch.empty(self.n, self.h, self.w, 3, device=dev, dtype=torch.uint8)
        status = torch.empty(self.n, device=dev, dtype=torch.int32)
        nbytes = lib.udh_png_workspace_bytes(self.plan.data_ptr())
        ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
        check(lib.udh_png_decode(self.plan.data_ptr(), _ptr(plan_d), _ptr(idat_d), _ptr(out), _ptr(status), int(bool(rgb)), _ptr(ws),
                                 nbytes, _stream()), "udh_png_decode")
        return out, status


def decode_png(blobs, h, w, rgb=False):
    """PNG files (bytes) the parser accepts, all h x w -> (uint8 [N,h,w,3] CUDA tensor, int32 [N] status): bit-identical to
    cv2.imread(..., IMREAD_COLOR) (BGR; RGB when rgb).  Raises UdhError naming the first file the device could not decode."""
    _lib.require_device()
    out, status = PngPlan(blobs, h, w).decode(rgb=rgb)
    st = status.cpu().numpy()
    bad = np.flatnonzero(st)
    if len(bad):
        raise _lib.UdhError("decode_png: image %d failed with status %d (%d of %d images failed)" % (bad[0], st[bad[0]], len(bad), len(st)))
    return out, status


# ------------------------------------------------------------------ baseline-JPEG encode
def encode_jpeg_device(imgs, quality=95):
    """uint8 CUDA tensor [N,h,w,3] (BGR) or [N,h,w] (gray) -> (out uint8 [N,cap], nbytes int64 [N], status int32 [N]) on the
    current stream: image k's file is out[k, :nbytes[k]]; nonzero status = that image failed."""
    _req(imgs, torch.uint8, "imgs")
    if imgs.dim() not in (3, 4) or (imgs.dim() == 4 and imgs.shape[3] != 3):
        raise _lib.UdhError("encode_jpeg: images must be [N,h,w,3] BGR or [N,h,w] gray (got %s)" % (tuple(imgs.shape),))
    n, h, w = imgs.shape[:3]
    ch = 3 if imgs.dim() == 4 else 1
    cap = lib.udh_jpeg_encode_capacity(h, w, ch)
    nb = lib.udh_jpeg_encode_workspace_bytes(max(n, 1), h, w, ch)
    if cap == 0 or nb == 0:
        raise _lib.UdhError("encode_jpeg: unsupported size %dx%d" % (h, w))
    out = torch.empty(n, cap, device=imgs.device, dtype=torch.uint8)
    nbytes = torch.empty(n, device=imgs.device, dtype=torch.int64)
    status = torch.empty(n, device=imgs.device, dtype=torch.int32)
    if n == 0:
        return out, nbytes, status
    ws = torch.empty(nb, device=imgs.device, dtype=torch.uint8)
    check(lib.udh_jpeg_encode(_ptr(imgs), n, h, w, ch, int(quality), _ptr(out), cap, _ptr(nbytes), _ptr(status), _ptr(ws), nb,
                              _stream()), "udh_jpeg_encode")
    return out, nbytes, status


def encode_jpeg(imgs, quality=95):
    """uint8 images [N,h,w,3] in cv2's BGR order or [N,h,w] gray (CUDA tensor, or anything torch.as_tensor takes) -> one
    JPEG file (bytes) per image, each byte-identical to cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, quality]).
    Raises UdhError naming the first image that could not be encoded."""
    _lib.require_device()
    t = torch.as_tensor(imgs)
    if not t.is_cuda:
        t = t.cuda()
    out, nbytes, status = encode_jpeg_device(t.contiguous(), quality)
    st = status.cpu().numpy()
    bad = np.flatnonzero(st)
    if len(bad):
        raise _lib.UdhError("encode_jpeg: image %d failed with status %d (%d of %d images failed)" % (bad[0], st[bad[0]], len(bad), len(st)))
    nb = nbytes.cpu().numpy()
    buf = out[:, :int(nb.max())].cpu().numpy() if len(nb) else None
    return [buf[k, :nb[k]].tobytes() for k in range(len(nb))]


# ------------------------------------------------------------------ report image of the test harnesses
def draw_report_u8(I_u8, Ip_u8, aug, verts, prime_left):
    """Decoded I, I' [B,h,w,3] uint8 (+ the [B,11] augmentation table or None) and the report's int32 vertices verts
    [B,20,2] (report.report_vertices) -> the report canvases [B,h,2w,3] uint8 as cv2 draws them: denorm(I') | denorm(I)
    when prime_left, else denorm(I) | denorm(I')."""
    _req(I_u8, torch.uint8, "I"); _req(Ip_u8, torch.uint8, "I_prime"); _req(verts, torch.int32, "verts")
    if aug is not None:
        _req(aug, torch.float32, "aug")
    if I_u8.dim() != 4 or I_u8.shape[3] != 3:
        raise _lib.UdhError("draw_report_u8: I must be [B,h,w,3] (got %s)" % (tuple(I_u8.shape),))
    B, Hh, W, _ = I_u8.shape
    if tuple(Ip_u8.shape) != tuple(I_u8.shape) or tuple(verts.shape) != (B, 20, 2) or (aug is not None and tuple(aug.shape) != (B, 11)):
        raise _lib.UdhError("draw_report_u8: I' must be shaped like I, verts [B,20,2] and aug [B,11] (got %s, %s, %s, %s)"
                            % (tuple(I_u8.shape), tuple(Ip_u8.shape), tuple(verts.shape), None if aug is None else tuple(aug.shape)))
    out = torch.empty(B, Hh, 2 * W, 3, device=I_u8.device, dtype=torch.uint8)
    nb = lib.udh_draw_report_workspace_bytes(B)
    ws = torch.empty(nb, device=I_u8.device, dtype=torch.uint8)
    check(lib.udh_draw_report_u8(_ptr(I_u8), _ptr(Ip_u8), _ptr(aug), int(bool(prime_left)), _ptr(verts), _ptr(out), _ptr(ws), nb,
                                 B, Hh, W, _stream()), "udh_draw_report_u8")
    return out


# ------------------------------------------------------------------ the dataset generator's warp
def gen_warp_u8(bgr, theta):
    """uint8 [N,h,w,3] CUDA tensor in cv2's BGR order, float64 theta [N,3,3] (CUDA, the generator's
    inv(M) inv(H_inverse) M) -> (gray [N,h,w], warped [N,h,w,3], warped_gray [N,h,w]): cv2.cvtColor(bgr, COLOR_RGB2GRAY) and
    the reference's numpy_transformer of the colour image and of the gray image, bit for bit."""
    _req(bgr, torch.uint8, "bgr"); _req(theta, torch.float64, "theta")
    if bgr.dim() != 4 or bgr.shape[3] != 3 or tuple(theta.shape) != (bgr.shape[0], 3, 3):
        raise _lib.UdhError("gen_warp_u8: bgr must be [N,h,w,3] and theta [N,3,3] (got %s and %s)" % (tuple(bgr.shape), tuple(theta.shape)))
    n, h, w, _ = bgr.shape
    gray = torch.empty(n, h, w, device=bgr.device, dtype=torch.uint8)
    warped = torch.empty_like(bgr)
    warped_gray = torch.empty_like(gray)
    check(lib.udh_gen_warp_u8(_ptr(bgr), _ptr(theta), n, h, w, _ptr(gray), _ptr(warped), _ptr(warped_gray), _stream()), "udh_gen_warp_u8")
    return gray, warped, warped_gray


def gray_u8(bgr):
    """uint8 [..., 3] CUDA tensor in cv2's BGR order -> uint8 [...]: cv2.cvtColor(bgr, COLOR_RGB2GRAY) as the reference
    calls it on BGR data, with gen_warp_u8's gray rule."""
    _req(bgr, torch.uint8, "bgr")
    if bgr.dim() < 1 or bgr.shape[-1] != 3:
        raise _lib.UdhError("gray_u8: bgr must be [..., 3] (got %s)" % (tuple(bgr.shape),))
    gray = torch.empty(bgr.shape[:-1], device=bgr.device, dtype=torch.uint8)
    check(lib.udh_gray_u8(_ptr(bgr), gray.numel(), _ptr(gray), _stream()), "udh_gray_u8")
    return gray


# ------------------------------------------------------------------ image alignment's warp
def warp_perspective_u8(src, M, dst_h, dst_w):
    """uint8 [B,h,w,C] CUDA tensor (C = 1 or 3, any channel order), float64 M [B,3,3] (CUDA) -> uint8 [B,dst_h,dst_w,C]:
    cv2.warpPerspective(src[b], M[b], (dst_w, dst_h)) per item (INTER_LINEAR, BORDER_CONSTANT 0), bit for bit."""
    _req(src, torch.uint8, "src")
    if src.dim() != 4 or src.shape[3] not in (1, 3):
        raise _lib.UdhError("warp_perspective_u8: src must be [B,h,w,1] or [B,h,w,3] (got %s)" % (tuple(src.shape),))
    B, h, w, C = src.shape
    M = M.reshape(-1, 9).contiguous()
    _req(M, torch.float64, "M")
    if M.shape[0] != B:
        raise _lib.UdhError("warp_perspective_u8: %d matrices for %d images" % (M.shape[0], B))
    out = torch.empty(B, int(dst_h), int(dst_w), C, device=src.device, dtype=torch.uint8)
    check(lib.udh_warp_perspective_u8(_ptr(src), _ptr(M), _ptr(out), B, h, w, C, int(dst_h), int(dst_w), _stream()),
          "udh_warp_perspective_u8")
    return out


# ------------------------------------------------------------------ sequence mosaic
def mosaic_tile_lists(M, sizes, dst_h, dst_w):
    """float64 M [n,3,3] (frame k -> canvas), sizes [(h_k, w_k)] -> udh_mosaic_blend_u8's CSR candidate lists (tile_ptr int32
    [ntiles + 1], tile_frames int32): per _lib.MOSAIC_TILE_H x MOSAIC_TILE_W canvas tile (row-major), the frames whose
    footprint can reach it, in frame order.  The footprint is the source rectangle grown by 1 px, corners (-1, -1) ..
    (w, h): when all four map with a positive denominator its image is a convex quad and the tiles meeting the quad's
    floor / ceil bounding box are listed; otherwise every tile is.  A valid pixel's source position lies within 1/64 px
    (rounding) of the frame, so the lists are conservative."""
    M = np.asarray(M, np.float64).reshape(-1, 3, 3)
    TH, TW = _lib.MOSAIC_TILE_H, _lib.MOSAIC_TILE_W
    gy, gx = -(-dst_h // TH), -(-dst_w // TW)
    tiles, frames = [], []
    for k, (h, w) in enumerate(sizes):
        p = np.array([[-1.0, -1.0, 1.0], [w, -1.0, 1.0], [w, h, 1.0], [-1.0, h, 1.0]]) @ M[k].T
        if np.isfinite(p).all() and (p[:, 2] > 0).all():
            x, y = p[:, 0] / p[:, 2], p[:, 1] / p[:, 2]
            if not (np.isfinite(x).all() and np.isfinite(y).all()):
                tx, ty = np.arange(gx), np.arange(gy)
            else:
                x0, x1 = max(np.floor(x.min()), 0.0), min(np.ceil(x.max()), dst_w - 1.0)
                y0, y1 = max(np.floor(y.min()), 0.0), min(np.ceil(y.max()), dst_h - 1.0)
                if x0 > x1 or y0 > y1:
                    continue
                tx = np.arange(int(x0) // TW, int(x1) // TW + 1)
                ty = np.arange(int(y0) // TH, int(y1) // TH + 1)
        else:
            tx, ty = np.arange(gx), np.arange(gy)
        ids = (ty[:, None] * gx + tx[None, :]).ravel()
        tiles.append(ids)
        frames.append(np.full(len(ids), k, np.int64))
    tiles = np.concatenate(tiles) if tiles else np.zeros(0, np.int64)
    frames = np.concatenate(frames) if frames else np.zeros(0, np.int64)
    if len(tiles) >= 2 ** 31:
        raise _lib.UdhError("mosaic_tile_lists: %d candidate entries do not fit int32" % len(tiles))
    order = np.lexsort((frames, tiles))
    ptr = np.zeros(gy * gx + 1, np.int64)
    ptr[1:] = np.cumsum(np.bincount(tiles, minlength=gy * gx))
    return ptr.astype(np.int32), frames[order].astype(np.int32)


def _gains(gains, n, dev, what):
    """Exposure gains [n], [n,1] or [n,3] (numpy or tensor) -> float64 [n,3] on dev (one gain repeated over the channels)."""
    g = (gains.detach().cpu().numpy() if isinstance(gains, torch.Tensor) else np.asarray(gains)).astype(np.float64)
    g = g.reshape(len(g), -1) if g.ndim else g.reshape(1, 1)
    if g.shape[0] != n or g.shape[1] not in (1, 3):
        raise _lib.UdhError("%s: gains must be [n], [n,1] or [n,3] for %d frames (got %s)" % (what, n, g.shape))
    return torch.from_numpy(np.broadcast_to(g, (n, 3)).copy()).to(dev)


def _mask_table(masks, rois, n, what):
    """Blend masks [n] (frame k's CUDA uint8 [roi_h,roi_w] on its multi-band ROI; ignored, may be None, where the ROI is
    empty) -> (host array of device pointers, rois int32 [n,4] with empty rows for the frames left out)."""
    masks = list(masks)
    if len(masks) != n:
        raise _lib.UdhError("%s: %d masks for %d frames" % (what, len(masks), n))
    rr = np.ascontiguousarray(np.asarray(rois, np.int64).astype(np.int32).reshape(n, 4))
    ptrs = (ctypes.c_void_p * max(n, 1))()
    for k, m in enumerate(masks):
        x0, y0, x1, y1 = (int(v) for v in rr[k])
        if x1 <= x0 or y1 <= y0:
            rr[k] = 0
            continue
        if m is None:
            raise _lib.UdhError("%s: frame %d meets the canvas but has no mask" % (what, k))
        _req(m, torch.uint8, "masks[%d]" % k)
        if tuple(m.shape) != (y1 - y0, x1 - x0):
            raise _lib.UdhError("%s: masks[%d] must be [%d,%d] (its ROI; got %s)" % (what, k, y1 - y0, x1 - x0, tuple(m.shape)))
        ptrs[k] = m.data_ptr()
    return ptrs, rr


def _frames_and_M(frames, M, what, channels):
    """frames (n CUDA uint8 tensors [h_k,w_k,C], or one [n,h,w,C] tensor) and M [n,3,3] (numpy or tensor) -> (frames as a
    list, M float64 [n,3,3] numpy, sizes [(h_k, w_k)]), checked: at least one frame, one matrix each, C in channels and the
    same for every frame."""
    frames = list(frames.unbind(0)) if isinstance(frames, torch.Tensor) else list(frames)
    Mh = (M.detach().cpu().numpy() if isinstance(M, torch.Tensor) else np.asarray(M)).astype(np.float64).reshape(-1, 3, 3)
    n = len(frames)
    if Mh.shape[0] != n:
        raise _lib.UdhError("%s: %d matrices for %d frames" % (what, Mh.shape[0], n))
    if n == 0:
        raise _lib.UdhError("%s: no frames" % what)
    for k, f in enumerate(frames):
        _req(f, torch.uint8, "frames[%d]" % k)
        if f.dim() != 3 or f.shape[2] not in channels or f.shape[2] != frames[0].shape[2]:
            raise _lib.UdhError("%s: frames must all be %s (frame %d is %s)"
                                % (what, " or all ".join("[h,w,%d]" % c for c in channels), k, tuple(f.shape)))
    return frames, Mh, [(int(f.shape[0]), int(f.shape[1])) for f in frames]


class _Fed(object):
    """frames and M (frame k -> canvas) as the multi-band blend takes them -> the frames it feeds, those whose ROI
    (mosaic.multiband_rois) meets the canvas, as the ROI entry points take them: n, dev, rois int64 [n,4], take (the fed
    frames' indices), m = len(take) and, when m > 0, frames [m], ptrs (host array of device pointers), sz int32 [m,2], rr
    int32 [m,4] (their ROIs) and M_d float64 [m,9] on the device (frame -> ROI)."""

    def __init__(self, frames, M, dst_h, dst_w, what, max_frames=None):
        from . import mosaic
        frames, Mh, sizes = _frames_and_M(frames, M, what, (3,))
        rois, Mr = mosaic.multiband_rois(Mh, sizes, int(dst_h), int(dst_w))
        self.n, self.dev, self.rois = len(frames), frames[0].device, rois
        self.take = [k for k in range(self.n) if rois[k, 2] > rois[k, 0] and rois[k, 3] > rois[k, 1]]
        m = self.m = len(self.take)
        if max_frames is not None and m > max_frames:
            raise _lib.UdhError("%s: %d frames meet the canvas (at most %d)" % (what, m, max_frames))
        if not m:
            return
        self.frames = [frames[k] for k in self.take]
        self.ptrs = (ctypes.c_void_p * m)(*[f.data_ptr() for f in self.frames])
        self.sz = np.ascontiguousarray(np.array([sizes[k] for k in self.take], np.int32).reshape(m, 2))
        self.rr = np.ascontiguousarray(rois[self.take].astype(np.int32))
        self.M_d = torch.from_numpy(np.ascontiguousarray(Mr[self.take].reshape(m, 9))).to(self.dev)

    def fed(self, items, what, name):
        """A per-frame list [n] -> its entries for the fed frames."""
        items = list(items)
        if len(items) != self.n:
            raise _lib.UdhError("%s: %d %s for %d frames" % (what, len(items), name, self.n))
        return [items[k] for k in self.take]


def mosaic_blend_u8(frames, M, dst_h, dst_w, feather, gains=None, masks=None, gain_maps=None):
    """frames: n CUDA uint8 tensors [h_k,w_k,C] (C = 1 or 3, sizes may differ; or one [n,h,w,C] tensor), M float64 [n,3,3]
    (frame k -> canvas; numpy or tensor) -> (mosaic uint8 [dst_h,dst_w,C], mask uint8 [dst_h,dst_w]): udh_mosaic_blend_u8's
    feathered blend of cv2.warpPerspective(frame k, M_k, (dst_w, dst_h)), bit for bit with oracle/mosaic.py.  The tile
    lists are built on the host (mosaic_tile_lists); the frames are read where they are.  gains ([n] or [n,3], e.g.
    mosaic_exposure_gains'): each frame's warp value is exposure-compensated first, saturate_u8(rint(v g)) in float64.
    masks ([n], e.g. mosaic_seam_masks' blend masks): frame k counts only where its mask, a CUDA uint8 [roi_h,roi_w] on its
    ROI (mosaic.multiband_rois), is set; a frame whose ROI misses the canvas takes None and counts nowhere.  gain_maps ([n],
    e.g. mosaic_exposure_gain_maps'; not with gains): each frame's warp value is compensated by its block gain map resized
    to its ROI, at the pixel's ROI coordinates, saturate_u8(rint(float32(v) g))."""
    from . import mosaic
    what = "mosaic_blend_u8"
    frames, Mh, sizes = _frames_and_M(frames, M, what, (1, 3))
    if gains is not None and gain_maps is not None:
        raise _lib.UdhError("%s: gains and gain_maps exclude each other" % what)
    n, C, dev = len(frames), frames[0].shape[2], frames[0].device
    ptr, idx = mosaic_tile_lists(Mh, sizes, int(dst_h), int(dst_w))
    ptr_d = torch.from_numpy(ptr).to(dev)
    idx_d = torch.from_numpy(idx if len(idx) else np.zeros(1, np.int32)).to(dev)
    M_d = torch.from_numpy(np.ascontiguousarray(Mh.reshape(n, 9))).to(dev)
    out = torch.empty(int(dst_h), int(dst_w), C, device=dev, dtype=torch.uint8)
    mask = torch.empty(int(dst_h), int(dst_w), device=dev, dtype=torch.uint8)
    nb = lib.udh_mosaic_workspace_bytes(n)
    ws = torch.empty(max(nb, 1), device=dev, dtype=torch.uint8)
    ptrs = (ctypes.c_void_p * n)(*[f.data_ptr() for f in frames])
    sz = np.ascontiguousarray(np.array(sizes, np.int32).reshape(n, 2))
    g_d = None if gains is None else _gains(gains, n, dev, what)
    gm = mp = rr = None
    if masks is not None or gain_maps is not None:
        rr = np.ascontiguousarray(mosaic.multiband_rois(Mh, sizes, int(dst_h), int(dst_w))[0].astype(np.int32))
    if gain_maps is not None:
        gm, _keep = _gain_map_table(gain_maps, rr, n, dev, what)
    if masks is not None:
        mp, rr = _mask_table(masks, rr, n, what)
    check(lib.udh_mosaic_blend_u8(ptrs, sz.ctypes.data, _ptr(M_d), _ptr(g_d), gm, mp, None if rr is None else rr.ctypes.data, n, C,
                                  _ptr(ptr_d), _ptr(idx_d), int(dst_h), int(dst_w), int(feather), _ptr(out), _ptr(mask), _ptr(ws), nb,
                                  _stream()), "udh_mosaic_blend_u8")
    return out, mask


def mosaic_multiband_u8(frames, M, dst_h, dst_w, bands, levels=False, gains=None, masks=None, gain_maps=None):
    """frames: n CUDA uint8 RGB tensors [h_k,w_k,3] (sizes may differ), M float64 [n,3,3] (frame k -> canvas; numpy or
    tensor) -> (mosaic uint8 [dst_h,dst_w,3], mask uint8 [dst_h,dst_w]): udh_mosaic_multiband_u8, byte for byte
    cv2.detail_MultiBandBlender(0, bands, CV_16S) fed each frame's warp on its ROI (oracle/multiband.py).  The ROIs and the
    frame -> ROI maps are formed on the host (mosaic.multiband_rois, which raises ValueError for a frame whose corners do not
    map to finite points with a positive denominator); a frame whose ROI misses the canvas is left out.  levels=True also
    returns the canvas pyramid as the feeds left it: [B' + 1] int16 CUDA tensors [Hp >> i, Wp >> i, 4] (acc, then wacc).
    gains ([n] or [n,3], e.g. mosaic_exposure_gains'): each ROI warp is exposure-compensated before it is fed,
    saturate_u8(rint(v g)) in float64, cv2's stitcher order.  masks ([n], e.g. mosaic_seam_masks' blend masks; None for a
    frame whose ROI misses the canvas): frame k is fed its mask, a CUDA uint8 [roi_h,roi_w], in place of its validity
    mask.  gain_maps ([n], e.g. mosaic_exposure_gain_maps'; not with gains): each ROI warp is compensated by its block gain
    map resized to the ROI, saturate_u8(rint(float32(v) g)), before it is fed."""
    what = "mosaic_multiband_u8"
    fed = _Fed(frames, M, dst_h, dst_w, what)
    if gains is not None and gain_maps is not None:
        raise _lib.UdhError("%s: gains and gain_maps exclude each other" % what)
    m, dev = fed.m, fed.dev
    out = torch.zeros(int(dst_h), int(dst_w), 3, device=dev, dtype=torch.uint8)
    mask = torch.zeros(int(dst_h), int(dst_w), device=dev, dtype=torch.uint8)
    g_d = None if gains is None else _gains(gains, fed.n, dev, what)
    if not m:
        return (out, mask, []) if levels else (out, mask)
    nb = lib.udh_mosaic_multiband_workspace_bytes(fed.rr.ctypes.data, m, int(dst_h), int(dst_w), int(bands))
    if nb == 0:
        raise _lib.UdhError("%s: bad arguments (%d frames, canvas %dx%d, %d bands)" % (what, m, dst_h, dst_w, bands))
    ws = torch.empty(nb, device=dev, dtype=torch.uint8)
    g_d = None if g_d is None else g_d[fed.take].contiguous()
    gm = mp = None
    if gain_maps is not None:
        gm, _keep = _gain_map_table(fed.fed(gain_maps, what, "gain maps"), fed.rr, m, dev, what)
    if masks is not None:
        mp, _ = _mask_table(fed.fed(masks, what, "masks"), fed.rr, m, what)
    check(lib.udh_mosaic_multiband_u8(fed.ptrs, fed.sz.ctypes.data, _ptr(fed.M_d), _ptr(g_d), gm, mp, fed.rr.ctypes.data, m, 3,
                                      int(dst_h), int(dst_w), int(bands), _ptr(out), _ptr(mask), _ptr(ws), nb, _stream()),
          "udh_mosaic_multiband_u8")
    if not levels:
        return out, mask
    off, dims = (ctypes.c_size_t * 11)(), (ctypes.c_int * 3)()
    check(lib.udh_debug_multiband_layout(fed.rr.ctypes.data, m, int(dst_h), int(dst_w), int(bands), off, dims),
          "udh_debug_multiband_layout")
    B, Hp, Wp = dims
    pyr = []
    for i in range(B + 1):
        cnt = (Hp >> i) * (Wp >> i) * 4
        pyr.append(ws[off[i]:off[i] + 2 * cnt].view(torch.int16).reshape(Hp >> i, Wp >> i, 4))
    return out, mask, pyr


# ------------------------------------------------------------------ exposure compensation
EXPOSURE_ALPHA, EXPOSURE_BETA = 0.01, 100.0       # cv2.detail.GainCompensator's weights of the gain and intensity terms


def roi_pairs(rois, diagonal):
    """rois [m,4] (x_lo, y_lo, x_hi, y_hi) -> CSR (pair_ptr int32 [m+1], pair_j int32 [P]) of the pairs whose rectangles
    intersect (cv2.detail.overlapRoi), row-major: i <= j with the diagonal (the exposure statistics' pairs), i < j without
    (cv2.detail.PairwiseSeamFinder's visiting order)."""
    r = np.asarray(rois, np.int64).reshape(-1, 4)
    x0, y0 = np.maximum(r[:, None, 0], r[None, :, 0]), np.maximum(r[:, None, 1], r[None, :, 1])
    x1, y1 = np.minimum(r[:, None, 2], r[None, :, 2]), np.minimum(r[:, None, 3], r[None, :, 3])
    hit = np.triu((x0 < x1) & (y0 < y1), 0 if diagonal else 1)
    ptr = np.zeros(len(r) + 1, np.int64)
    ptr[1:] = np.cumsum(hit.sum(1))
    return ptr.astype(np.int32), np.nonzero(hit)[1].astype(np.int32)


def exposure_norm_sum(l0, l1, l2):
    """The three 21-bit limb sums of udh_mosaic_exposure_stats_u8's sum q (q = norm 2^52, an integer) -> sum norm: the exact
    total, rounded to double once (ties to even).  Scalars give a float; arrays, elementwise, a float64 array."""
    if np.ndim(l0):
        return np.array([exposure_norm_sum(*v) for v in zip(l0, l1, l2)], np.float64)
    return math.ldexp(float(int(l0) + (int(l1) << 21) + (int(l2) << 42)), -52)


class _ExposureStats(_Fed):
    """udh_mosaic_exposure_stats_u8 on fixed frames: the device-side frame table, pairs and output, reused by every feed."""

    def __init__(self, frames, M, dst_h, dst_w):
        _Fed.__init__(self, frames, M, dst_h, dst_w, "mosaic_exposure_stats", _lib.EXPOSURE_MAX_FRAMES)
        self.dst = (int(dst_h), int(dst_w))
        m = self.m
        if not m:
            self.i = self.j = np.zeros(0, np.int64)
            return
        ptr, pj = roi_pairs(self.rr, True)
        self.i = np.repeat(np.arange(m), np.diff(ptr)).astype(np.int64)
        self.j = pj.astype(np.int64)
        self.ptr_d, self.pj_d = torch.from_numpy(ptr).to(self.dev), torch.from_numpy(pj).to(self.dev)
        self.out = torch.empty(len(pj), _lib.EXPOSURE_STATS, device=self.dev, dtype=torch.int64)
        self.nb = lib.udh_mosaic_exposure_workspace_bytes(m)
        self.ws = torch.empty(max(self.nb, 1), device=self.dev, dtype=torch.uint8)

    def __call__(self, history=None, norms=True):
        """history: None or float64 [t,m,3] (the fed frames' gains of feeds 0..t-1) -> uint64 [P,13] numpy."""
        if not self.m:
            return np.zeros((0, _lib.EXPOSURE_STATS), np.uint64)
        t = 0 if history is None else int(np.asarray(history).shape[0])
        h_d = None
        if t:
            h_d = torch.from_numpy(np.ascontiguousarray(np.asarray(history, np.float64).reshape(t, self.m, 3))).to(self.dev)
        check(lib.udh_mosaic_exposure_stats_u8(self.ptrs, self.sz.ctypes.data, _ptr(self.M_d), self.rr.ctypes.data, self.m,
                                               _ptr(self.ptr_d), _ptr(self.pj_d), len(self.j), _ptr(h_d) if t else None, t,
                                               int(bool(norms)), self.dst[0], self.dst[1], _ptr(self.out), _ptr(self.ws), self.nb,
                                               _stream()), "udh_mosaic_exposure_stats_u8")
        return self.out.cpu().numpy().view(np.uint64)


def mosaic_exposure_stats(frames, M, dst_h, dst_w, history=None, norms=True):
    """The exposure compensators' pair statistics of the frames' ROI warps (udh_mosaic_exposure_stats_u8), for tests and
    tools.  frames, M as mosaic_multiband_u8 takes them; history None or [t,m,3] over the fed frames.  -> dict(take (the fed
    frames: those whose ROI meets the canvas), i, j [P] (pairs of fed-frame indices, i <= j, ROIs intersecting), count
    int64 [P], sums int64 [P,2,3] (frame i's, frame j's channel sums), norms float64 [P,2] (sum of cv2's norm(Vec3b),
    exact and rounded once; 0 without norms), raw uint64 [P,13])."""
    st = _ExposureStats(frames, M, dst_h, dst_w)
    raw = st(history, norms)
    ns = np.stack([exposure_norm_sum(*raw[:, 7:10].T), exposure_norm_sum(*raw[:, 10:13].T)], 1)
    return dict(take=st.take, i=st.i, j=st.j, count=raw[:, 0].astype(np.int64), sums=raw[:, 1:7].astype(np.int64).reshape(-1, 2, 3),
                norms=ns, raw=raw)


def exposure_solve(m, i, j, count, Isum_i, Isum_j):
    """One feed of cv2.detail.GainCompensator on m images from its pair statistics (pairs i <= j whose ROIs intersect,
    their mask-intersection counts and the two sums) -> gains float64 [m].  N_ij = N_ji = max(1, count); where count > 0,
    I_ij = Isum_i / N_ij and I_ji = Isum_j / N_ij, and an off-diagonal pair keeps both frames from being skipped.  Over the
    unskipped frames in order: b_i += beta N_ij, A_ii += beta N_ij and, for j != i, A_ii += 2 alpha I_ij^2 N_ij,
    A_ij -= 2 alpha I_ij I_ji N_ij; gains = cv2.solve(A, b) (LU) there, 1 for skipped frames.  The sums are formed in
    cv2's order, so equal statistics give cv2's bits."""
    import cv2
    N = np.zeros((m, m), np.int64)
    I = np.zeros((m, m), np.float64)
    skip = np.ones(m, bool)
    for a, b, c, s1, s2 in zip(i, j, count, Isum_i, Isum_j):
        a, b = int(a), int(b)
        N[a, b] = N[b, a] = max(1, int(c))
        if c == 0:
            continue
        if a != b:
            skip[a] = skip[b] = False
        I[a, b] = float(s1) / N[a, b]
        I[b, a] = float(s2) / N[a, b]
    g = np.ones(m, np.float64)
    idx = [k for k in range(m) if not skip[k]]
    if not idx:
        return g
    A = np.zeros((len(idx), len(idx)), np.float64)
    rhs = np.zeros((len(idx), 1), np.float64)
    al, be = EXPOSURE_ALPHA, EXPOSURE_BETA
    for ki, a in enumerate(idx):
        for kj, b in enumerate(idx):
            nab, iab, iba = int(N[a, b]), float(I[a, b]), float(I[b, a])
            rhs[ki, 0] += be * nab
            A[ki, ki] += be * nab
            if b != a:
                A[ki, ki] += 2 * al * iab * iab * nab
                A[ki, kj] -= 2 * al * iab * iba * nab
    _, x = cv2.solve(A, rhs)
    g[idx] = x.reshape(-1)
    return g


def mosaic_exposure_gains(frames, M, dst_h, dst_w, mode="gain", feeds=1):
    """frames: n CUDA uint8 RGB tensors [h_k,w_k,3], M float64 [n,3,3] (frame k -> canvas) -> gains float64 [n,3]: what
    cv2.detail_GainCompensator(feeds) (mode "gain": one gain per frame, repeated over the channels) or
    cv2.detail_ChannelsCompensator(feeds) ("channels": one per channel) computes when fed the multi-band blend's inputs
    (each frame's ROI warp, its validity mask and the ROI's top-left; oracle/exposure.py).  A frame whose ROI misses the
    canvas is not fed and gets 1.  Feed t sees the images compensated by feeds 0..t-1 in turn; the gains are the product
    of the feeds'.  The pair statistics come from udh_mosaic_exposure_stats_u8 (exact integer sums; in "gain" mode the sums
    of norms are exact and rounded once where cv2 adds in row order, so the gains agree to cv2's own summation error; in
    "channels" mode they are cv2's bits); the small system is solved on the host."""
    if mode not in ("gain", "channels"):
        raise ValueError("mode must be 'gain' or 'channels' (got %r)" % (mode,))
    if not 1 <= int(feeds) <= _lib.EXPOSURE_MAX_FEEDS:
        raise ValueError("feeds must be in 1..%d (got %r)" % (_lib.EXPOSURE_MAX_FEEDS, feeds))
    st = _ExposureStats(frames, M, dst_h, dst_w)
    gains = np.ones((st.n, 3), np.float64)
    if not st.m:
        return gains
    hist, acc = [], None
    for _ in range(int(feeds)):
        raw = st(np.stack(hist) if hist else None, norms=mode == "gain")
        count = raw[:, 0].astype(np.int64)
        if mode == "gain":
            g = exposure_solve(st.m, st.i, st.j, count, exposure_norm_sum(*raw[:, 7:10].T), exposure_norm_sum(*raw[:, 10:13].T))
            g3 = np.repeat(g[:, None], 3, 1)
        else:
            g3 = np.stack([exposure_solve(st.m, st.i, st.j, count, raw[:, 1 + c].astype(np.int64),
                                          raw[:, 4 + c].astype(np.int64)) for c in range(3)], 1)
        acc = g3.copy() if acc is None else acc * g3
        hist.append(g3)
    gains[st.take] = acc
    return gains


# ------------------------------------------------------------------ block exposure compensation
EXPOSURE_BLOCK_TOL, EXPOSURE_BLOCK_MAX_ITER = 1e-15, 2000  # udh_exposure_block_solve's stop: |r| <= tol |b|


def exposure_block_grid(rois, block):
    """rois [m,4] (x_lo, y_lo, x_hi, y_hi), block side -> (blocks int32 [m,4]: bw, bh, bpx, bpy; boff int64 [m+1]): cv2's
    BlocksCompensator blocks of each ROI (bpx = ceil(roi_w / block), bw = ceil(roi_w / bpx), likewise in y), numbered
    frame-major, then row-major, frame k's from boff[k]."""
    r = np.asarray(rois, np.int64).reshape(-1, 4)
    w, h = r[:, 2] - r[:, 0], r[:, 3] - r[:, 1]
    bpx, bpy = -(-w // int(block)), -(-h // int(block))
    bw, bh = -(-w // bpx), -(-h // bpy)
    if ((bpx - 1) * bw >= w).any() or ((bpy - 1) * bh >= h).any():
        raise _lib.UdhError("exposure_block_grid: a %d-px block leaves an empty block in a ROI" % block)
    boff = np.zeros(len(r) + 1, np.int64)
    boff[1:] = np.cumsum(bpx * bpy)
    if boff[-1] > _lib.EXPOSURE_MAX_BLOCKS:
        raise _lib.UdhError("exposure_block_grid: %d blocks (at most %d)" % (boff[-1], _lib.EXPOSURE_MAX_BLOCKS))
    return np.stack([bw, bh, bpx, bpy], 1).astype(np.int32), boff


def _block_axis(ra, ea, bwa, rb, eb, bwb, lo, hi):
    """One axis of a frame pair: block intervals [r + i bw, min(r + (i + 1) bw, e)) of both frames over [lo, hi) -> (i_a, i_b,
    cell) of every intersecting pair of intervals, the number of cells, and the first blocks i_a0, i_b0."""
    a0, a1 = (lo - ra) // bwa, (hi - 1 - ra) // bwa
    b0, b1 = (lo - rb) // bwb, (hi - 1 - rb) // bwb
    ia, ib = np.arange(a0, a1 + 1), np.arange(b0, b1 + 1)
    x0 = np.maximum(ra + ia[:, None] * bwa, rb + ib[None, :] * bwb)
    x1 = np.minimum(np.minimum(ra + (ia[:, None] + 1) * bwa, ea), np.minimum(rb + (ib[None, :] + 1) * bwb, eb))
    hit = np.nonzero(x0 < x1)
    return ia[hit[0]], ib[hit[1]], hit[0] + hit[1], (a1 - a0) + (b1 - b0) + 1


def exposure_block_cells(rois, blocks, boff):
    """The block pairs of cv2's block compensator and where udh_mosaic_exposure_block_stats_u8 sums them.  -> dict(pair_ptr,
    pair_j (the frame pairs i <= j whose ROIs intersect, roi_pairs), cell_off int64 [P], cell_nx int32 [P], nslots,
    a, b int64 [Q] (every pair of blocks a <= b whose rectangles intersect, a block with itself included), slot int64 [Q])."""
    r = np.asarray(rois, np.int64).reshape(-1, 4)
    ptr, pj = roi_pairs(r, True)
    P = len(pj)
    cell_off, cell_nx = np.zeros(P, np.int64), np.zeros(P, np.int32)
    A, B, S = [], [], []
    o, p = 0, 0
    for i in range(len(r)):
        for j in pj[ptr[i]:ptr[i + 1]]:
            bw_i, bh_i, bpx_i, _ = (int(v) for v in blocks[i])
            bw_j, bh_j, bpx_j, _ = (int(v) for v in blocks[j])
            x0, y0 = max(r[i, 0], r[j, 0]), max(r[i, 1], r[j, 1])
            x1, y1 = min(r[i, 2], r[j, 2]), min(r[i, 3], r[j, 3])
            xa, xb, cx, nx = _block_axis(r[i, 0], r[i, 2], bw_i, r[j, 0], r[j, 2], bw_j, x0, x1)
            ya, yb, cy, ny = _block_axis(r[i, 1], r[i, 3], bh_i, r[j, 1], r[j, 3], bh_j, y0, y1)
            cell_off[p], cell_nx[p] = o, nx
            A.append((boff[i] + ya[:, None] * bpx_i + xa[None, :]).ravel())
            B.append((boff[j] + yb[:, None] * bpx_j + xb[None, :]).ravel())
            S.append((o + cy[:, None] * nx + cx[None, :]).ravel())
            o += nx * ny
            p += 1
    return dict(pair_ptr=ptr, pair_j=pj, cell_off=cell_off, cell_nx=cell_nx, nslots=o, a=np.concatenate(A).astype(np.int64),
                b=np.concatenate(B).astype(np.int64), slot=np.concatenate(S).astype(np.int64))


def exposure_block_system(nblocks, a, b, count, sum_a, sum_b):
    """One feed of cv2.detail.GainCompensator over the blocks as a sparse system: block pairs a <= b whose rectangles
    intersect (each block with itself included), their counts and sums -> (keep int64 [n] (the unskipped blocks, in order),
    CSR row_ptr int32 [n+1], col int32, val float64, rhs float64 [n]).  The rule is exposure_solve's: N = max(1, count),
    I_ab = sum_a / N and I_ba = sum_b / N where count > 0, a block is skipped unless it has a positive-count pair with
    another block, and over the unskipped blocks, for row i and j ascending: b_i += beta N_ij, A_ii += beta N_ij and, for
    j != i, A_ii += 2 alpha I_ij^2 N_ij, A_ij -= 2 alpha I_ij I_ji N_ij, in that order, so A and b equal cv2's dense ones bit
    for bit (pairs whose rectangles do not intersect add nothing)."""
    a, b, count = (np.asarray(v, np.int64) for v in (a, b, count))
    N = np.maximum(count, 1).astype(np.float64)
    pos, off = count > 0, a != b
    Iab = np.where(pos, np.asarray(sum_a, np.float64) / N, 0.0)
    Iba = np.where(pos, np.asarray(sum_b, np.float64) / N, 0.0)
    skip = np.ones(int(nblocks), bool)
    skip[a[pos & off]] = False
    skip[b[pos & off]] = False
    keep = np.flatnonzero(~skip)
    idx = np.full(int(nblocks), -1, np.int64)
    idx[keep] = np.arange(len(keep))
    use = ~skip[a] & ~skip[b]
    u2 = use & off
    row = np.concatenate([idx[a[use]], idx[b[u2]]])
    col = np.concatenate([idx[b[use]], idx[a[u2]]])
    n_e = np.concatenate([N[use], N[u2]])
    i_rc = np.concatenate([Iab[use], Iba[u2]])
    i_cr = np.concatenate([Iba[use], Iab[u2]])
    order = np.lexsort((col, row))
    row, col, n_e, i_rc, i_cr = row[order], col[order], n_e[order], i_rc[order], i_cr[order]
    n = len(keep)
    ptr = np.zeros(n + 1, np.int64)
    ptr[1:] = np.cumsum(np.bincount(row, minlength=n))
    k_in_row = np.arange(len(row)) - ptr[row]
    al, be = EXPOSURE_ALPHA, EXPOSURE_BETA
    diag, rhs = np.zeros(n), np.zeros(n)
    nd = col != row
    val = np.where(nd, 0.0 - 2 * al * i_rc * i_cr * n_e, 0.0)
    by_k = np.argsort(k_in_row, kind="stable")
    bounds = np.searchsorted(k_in_row[by_k], np.arange(int(k_in_row.max(initial=-1)) + 2))
    for k in range(len(bounds) - 1):
        e = by_k[bounds[k]:bounds[k + 1]]                   # one entry per row: the k-th of each row
        rr = row[e]
        rhs[rr] += be * n_e[e]
        diag[rr] += be * n_e[e]
        e2 = e[nd[e]]
        diag[row[e2]] += 2 * al * i_rc[e2] * i_rc[e2] * n_e[e2]
    val[~nd] = diag[row[~nd]]
    return keep, ptr.astype(np.int32), col.astype(np.int32), val, rhs


def exposure_block_solve(row_ptr, col, val, rhs, dev, tol=EXPOSURE_BLOCK_TOL, max_iter=EXPOSURE_BLOCK_MAX_ITER):
    """udh_exposure_block_solve on the device dev -> (x float64 [n] numpy, iterations, final |r| / |b|)."""
    n = len(rhs)
    t = [torch.from_numpy(np.ascontiguousarray(v)).to(dev) for v in (row_ptr, col, val, rhs)]
    x = torch.empty(n, device=dev, dtype=torch.float64)
    info = torch.zeros(2, device=dev, dtype=torch.int64)
    nb = lib.udh_exposure_block_solve_workspace_bytes(n)
    ws = torch.empty(max(nb, 1), device=dev, dtype=torch.uint8)
    check(lib.udh_exposure_block_solve(n, _ptr(t[0]), _ptr(t[1]), _ptr(t[2]), _ptr(t[3]), float(tol), int(max_iter), _ptr(x), _ptr(info),
                                       _ptr(ws), nb, _stream()), "udh_exposure_block_solve")
    inf = info.cpu().numpy()
    return x.cpu().numpy(), int(inf[0]), float(inf[1:2].view(np.float64)[0])


class _ExposureBlockStats(_Fed):
    """udh_mosaic_exposure_block_stats_u8 on fixed frames and blocks: tables, cells and output, reused by every feed."""

    def __init__(self, frames, M, dst_h, dst_w, block):
        if int(block) < 1:
            raise ValueError("block must be >= 1 (got %r)" % (block,))
        _Fed.__init__(self, frames, M, dst_h, dst_w, "mosaic_exposure_gain_maps", _lib.EXPOSURE_MAX_FRAMES)
        self.dst = (int(dst_h), int(dst_w))
        m, dev = self.m, self.dev
        if not m:
            return
        self.blocks, boff = exposure_block_grid(self.rr, block)
        self.blocks = np.ascontiguousarray(self.blocks)
        self.boff, self.nblocks = np.ascontiguousarray(boff[:-1]), int(boff[-1])
        c = self.cells = exposure_block_cells(self.rr, self.blocks, boff)
        self.ptr_d, self.pj_d = torch.from_numpy(c["pair_ptr"]).to(dev), torch.from_numpy(c["pair_j"]).to(dev)
        self.off_d, self.nx_d = torch.from_numpy(c["cell_off"]).to(dev), torch.from_numpy(c["cell_nx"]).to(dev)
        self.slot_d = torch.from_numpy(c["slot"]).to(dev)
        self.out = torch.empty(c["nslots"], _lib.EXPOSURE_STATS, device=dev, dtype=torch.int64)
        self.nb = lib.udh_mosaic_exposure_block_workspace_bytes(m)
        self.ws = torch.empty(max(self.nb, 1), device=dev, dtype=torch.uint8)

    def __call__(self, history=None, norms=True):
        """history: None or a CUDA float64 [t,nblocks,3] -> uint64 [Q,13] numpy, the statistics of cells['a'], cells['b']."""
        t = 0 if history is None else int(history.shape[0])
        c = self.cells
        check(lib.udh_mosaic_exposure_block_stats_u8(self.ptrs, self.sz.ctypes.data, _ptr(self.M_d), self.rr.ctypes.data, self.m,
                                                     self.blocks.ctypes.data, self.boff.ctypes.data, self.nblocks, _ptr(self.ptr_d),
                                                     _ptr(self.pj_d), len(c["pair_j"]), _ptr(self.off_d), _ptr(self.nx_d), c["nslots"],
                                                     _ptr(history) if t else None, t, int(bool(norms)), self.dst[0], self.dst[1],
                                                     _ptr(self.out), _ptr(self.ws), self.nb, _stream()),
              "udh_mosaic_exposure_block_stats_u8")
        return self.out.index_select(0, self.slot_d).cpu().numpy().view(np.uint64)


def mosaic_exposure_block_stats(frames, M, dst_h, dst_w, block=32, history=None, norms=True):
    """The block compensators' block-pair statistics of the frames' ROI warps (udh_mosaic_exposure_block_stats_u8), for
    tests and tools.  history None or float64 [t,nblocks,3].  -> dict(take, blocks, boff, a, b [Q] (block pairs a <= b whose
    rectangles intersect), count int64 [Q], sums int64 [Q,2,3], norms float64 [Q,2] (0 without norms))."""
    st = _ExposureBlockStats(frames, M, dst_h, dst_w, block)
    if not st.m:
        return dict(take=[], a=np.zeros(0, np.int64), b=np.zeros(0, np.int64))
    h = None if history is None else torch.from_numpy(np.ascontiguousarray(history, np.float64)).to(st.dev)
    raw = st(h, norms)
    return dict(take=st.take, blocks=st.blocks, boff=st.boff, a=st.cells["a"], b=st.cells["b"], count=raw[:, 0].astype(np.int64),
                sums=raw[:, 1:7].astype(np.int64).reshape(-1, 2, 3),
                norms=np.stack([exposure_norm_sum(*raw[:, 7:10].T), exposure_norm_sum(*raw[:, 10:13].T)], 1), raw=raw)


def mosaic_exposure_block_gains(frames, M, dst_h, dst_w, mode="gain", feeds=1, block=32):
    """mosaic_exposure_gain_maps with its working: -> dict(take, maps [n] (None where not fed), gains float64 [nblocks,3]
    (the blocks' unfiltered gains, the product of the feeds'), blocks, boff, unknowns [per feed and system], iters,
    residual)."""
    if mode not in ("gain", "channels"):
        raise ValueError("mode must be 'gain' or 'channels' (got %r)" % (mode,))
    if not 1 <= int(feeds) <= _lib.EXPOSURE_MAX_FEEDS:
        raise ValueError("feeds must be in 1..%d (got %r)" % (_lib.EXPOSURE_MAX_FEEDS, feeds))
    st = _ExposureBlockStats(frames, M, dst_h, dst_w, block)
    out = dict(take=st.take, maps=[None] * st.n, unknowns=[], iters=[], residual=[])
    if not st.m:
        return out
    nbk, c = st.nblocks, st.cells
    hist = torch.empty(int(feeds), nbk, 3, device=st.dev, dtype=torch.float64)
    acc = None
    for t in range(int(feeds)):
        raw = st(hist[:t] if t else None, norms=mode == "gain")
        count = raw[:, 0].astype(np.int64)
        if mode == "gain":
            pos = (count > 0) & (c["a"] != c["b"])              # a block's own mean never enters the system
            sa, sb = np.zeros(len(count)), np.zeros(len(count))
            sa[pos], sb[pos] = exposure_norm_sum(*raw[pos, 7:10].T), exposure_norm_sum(*raw[pos, 10:13].T)
            sums = [(sa, sb)]
        else:
            sums = [(raw[:, 1 + ch].astype(np.int64), raw[:, 4 + ch].astype(np.int64)) for ch in range(3)]
        g3 = np.ones((nbk, 3), np.float64)
        for ch, (sa, sb) in enumerate(sums):
            keep, ptr, col, val, rhs = exposure_block_system(nbk, c["a"], c["b"], count, sa, sb)
            out["unknowns"].append(len(keep))
            if not len(keep):
                continue
            x, it, res = exposure_block_solve(ptr, col, val, rhs, st.dev)
            out["iters"].append(it)
            out["residual"].append(res)
            if mode == "gain":
                g3[keep] = x[:, None]
            else:
                g3[keep, ch] = x
        acc = g3.copy() if acc is None else acc * g3
        hist[t] = torch.from_numpy(g3).to(st.dev)
    ch = 1 if mode == "gain" else 3
    g_d = torch.from_numpy(acc).to(st.dev)
    maps = torch.empty(nbk * ch, device=st.dev, dtype=torch.float32)
    nb = lib.udh_exposure_gain_maps_workspace_bytes(nbk, ch)
    ws = torch.empty(nb, device=st.dev, dtype=torch.uint8)
    check(lib.udh_exposure_gain_maps(_ptr(g_d), st.m, st.blocks.ctypes.data, st.boff.ctypes.data, nbk, ch, _ptr(maps), _ptr(ws), nb,
                                     _stream()), "udh_exposure_gain_maps")
    for q, k in enumerate(st.take):
        bpx, bpy = int(st.blocks[q, 2]), int(st.blocks[q, 3])
        o = int(st.boff[q]) * ch
        mp = maps[o:o + bpx * bpy * ch]
        out["maps"][k] = mp.view(bpy, bpx) if ch == 1 else mp.view(bpy, bpx, 3)
    out.update(gains=acc, blocks=st.blocks, boff=st.boff)
    return out


def mosaic_exposure_gain_maps(frames, M, dst_h, dst_w, mode="gain", feeds=1, block=32):
    """frames: n CUDA uint8 RGB tensors [h_k,w_k,3], M float64 [n,3,3] (frame k -> canvas) -> per frame its gain map, a CUDA
    float32 [bpy,bpx] ("gain") or [bpy,bpx,3] ("channels") tensor (None for a frame whose ROI misses the canvas): what
    cv2.detail_BlocksGainCompensator(block, block, feeds) / BlocksChannelsCompensator's getMatGains() gives when fed the
    multi-band blend's inputs (oracle/exposure_blocks.py).  Each ROI warp is cut into blocks of about block x block px;
    udh_mosaic_exposure_block_stats_u8 sums every block pair's statistics exactly, the sparse system is assembled on the
    host in cv2's order (exposure_block_system) and solved on the GPU by conjugate gradients (udh_exposure_block_solve, to
    |r| <= 1e-15 |b|), and udh_exposure_gain_maps filters the float32 maps as cv2 does.  The blends apply them with
    gain_maps=."""
    return mosaic_exposure_block_gains(frames, M, dst_h, dst_w, mode, feeds, block)["maps"]


def map_taps(n, N):
    """The resize taps of a map axis of n -> an ROI axis of N (udh_map_tap [N] as int32 [N,4]: s0, s1, and the float32
    weights' bits): generic INTER_LINEAR in float32 (oracle/exposure_blocks.resize_map)."""
    if n == N:
        s = np.arange(N)
        f = np.zeros(N, np.float32)
    else:
        f = ((np.arange(N) + 0.5) * (1.0 / (float(N) / float(n))) - 0.5).astype(np.float32)
        s = np.floor(f).astype(np.int64)
        f = (f - s.astype(np.float32)).astype(np.float32)
        f[(s < 0) | (s >= n - 1)] = 0
        s = np.clip(s, 0, n - 1)
    t = np.zeros((N, 4), np.int32)
    t[:, 0], t[:, 1] = s, np.minimum(s + 1, n - 1)
    t[:, 2] = (np.float32(1) - f).astype(np.float32).view(np.int32)
    t[:, 3] = f.view(np.int32)
    return t


def _gain_map_table(gain_maps, rois, n, dev, what):
    """Per-frame gain maps (CUDA float32 [bpy,bpx(,3)], None where the ROI is empty) on rois [n,4] -> (udh_gain_map [n],
    the tensors it points to)."""
    gain_maps = list(gain_maps)
    if len(gain_maps) != n:
        raise _lib.UdhError("%s: %d gain maps for %d frames" % (what, len(gain_maps), n))
    table = (_lib.GainMap * n)()
    keep = []
    for k, mp in enumerate(gain_maps):
        x0, y0, x1, y1 = (int(v) for v in rois[k])
        if x1 <= x0 or y1 <= y0:
            continue
        if mp is None:
            raise _lib.UdhError("%s: frame %d meets the canvas but has no gain map" % (what, k))
        _req(mp, torch.float32, "gain_maps[%d]" % k)
        if mp.dim() not in (2, 3) or (mp.dim() == 3 and mp.shape[2] != 3) or not mp.is_contiguous():
            raise _lib.UdhError("%s: gain_maps[%d] must be a contiguous [bpy,bpx] or [bpy,bpx,3] (got %s)" % (what, k, tuple(mp.shape)))
        cols = torch.from_numpy(map_taps(mp.shape[1], x1 - x0)).to(dev)
        rows = torch.from_numpy(map_taps(mp.shape[0], y1 - y0)).to(dev)
        keep += [mp, cols, rows]
        table[k] = _lib.GainMap(mp.data_ptr(), cols.data_ptr(), rows.data_ptr(), int(mp.shape[1]), int(mp.shape[0]),
                                1 if mp.dim() == 2 else 3, 0)
    return table, keep


# ------------------------------------------------------------------ seam finding
SEAM_FINDERS = ("voronoi", "gc_color")


def mosaic_seam_masks(frames, M, dst_h, dst_w, finder="voronoi", scale=1.0):
    """frames: n CUDA uint8 RGB tensors [h_k,w_k,3], M float64 [n,3,3] (frame k -> canvas) -> dict(take (the fed frames:
    those whose ROI meets the canvas), rois int64 [n,4] (mosaic.multiband_rois), seam [m], blend [m]): per fed frame its
    seam mask and blend mask, CUDA uint8 [roi_h,roi_w] (0 / 255), and cv2.dilate of that AND the validity, the mask cv2's
    stitcher feeds its blender.  finder "voronoi": byte for byte what cv2.detail's Voronoi seam finder leaves in the
    multi-band blend's validity masks (udh_mosaic_seam_masks_u8; oracle/seam.py states the rule).  A frame lying inside
    another one's seam region vanishes (an all-zero mask), as in cv2.  finder "gc_color": cv2.detail's
    GraphCutSeamFinder(COST_COLOR) on the uncompensated ROI warps, as the canonical minimum cut of each pair's window
    (udh_mosaic_seam_gc_masks_u8; oracle/seam_gc.py states the rule), with cut int64 [pairs]: each pair's cut value, the
    pairs in cv2's visiting order.
    scale a < 1 (mosaic.seam_scale: cv2's seam_megapix) finds the seams at reduced resolution (oracle/seam_scale.py): the
    frames resized by a (resize_linear_exact_u8), the finder on mosaic.seam_geometry's maps and seam canvas, and each seam
    mask upscaled to the full ROI (udh_mosaic_seam_upscale_u8): blend [m] on the full ROIs, graded (1 .. 254 along the
    seams), seam [m] each fed frame's seam mask on its seam ROI ([0,0] where that misses the seam canvas), seam_rois int64
    [n,4] and scale; cut is the seam-scale finder's."""
    if finder not in SEAM_FINDERS:
        raise ValueError("finder must be one of %s (got %r)" % (", ".join(SEAM_FINDERS), finder))
    if not 0.0 < float(scale) <= 1.0:
        raise ValueError("scale must be in (0, 1] (got %r)" % (scale,))
    if float(scale) < 1.0:
        return _scaled_seam_masks(frames, M, dst_h, dst_w, finder, float(scale))
    gc = finder == "gc_color"
    fed = _Fed(frames, M, dst_h, dst_w, "mosaic_seam_masks", _lib.EXPOSURE_MAX_FRAMES)
    out = dict(take=fed.take, rois=fed.rois, seam=[], blend=[])
    if gc:
        out["cut"] = np.zeros(0, np.int64)
    if not fed.m:
        return out
    m, dev, rr = fed.m, fed.dev, fed.rr
    ptr, pj = roi_pairs(rr, False)
    npairs = int(ptr[-1])
    pj = pj if len(pj) else np.zeros(1, np.int32)
    hw = np.stack([rr[:, 3] - rr[:, 1], rr[:, 2] - rr[:, 0]], 1).astype(np.int64)
    off = np.concatenate([[0], np.cumsum(hw[:, 0] * hw[:, 1])])
    seam = torch.empty(int(off[-1]), device=dev, dtype=torch.uint8)
    blend = torch.empty(int(off[-1]), device=dev, dtype=torch.uint8)
    name = "udh_mosaic_seam_gc_masks_u8" if gc else "udh_mosaic_seam_masks_u8"
    ws_bytes = lib.udh_mosaic_seam_gc_workspace_bytes if gc else lib.udh_mosaic_seam_workspace_bytes
    nb = ws_bytes(rr.ctypes.data, m, ptr.ctypes.data, pj.ctypes.data, int(dst_h), int(dst_w))
    if nb == 0:
        raise _lib.UdhError("mosaic_seam_masks: bad arguments (%d frames, canvas %dx%d)" % (m, dst_h, dst_w))
    ws = torch.empty(nb, device=dev, dtype=torch.uint8)
    args = (fed.ptrs, fed.sz.ctypes.data, _ptr(fed.M_d), rr.ctypes.data, m, ptr.ctypes.data, pj.ctypes.data, int(dst_h), int(dst_w),
            _ptr(seam), _ptr(blend))
    if gc:
        cut = np.zeros(max(npairs, 1), np.int64)
        check(lib.udh_mosaic_seam_gc_masks_u8(*args, cut.ctypes.data, _ptr(ws), nb, _stream()), name)
        out["cut"] = cut[:npairs]
    else:
        check(lib.udh_mosaic_seam_masks_u8(*args, _ptr(ws), nb, _stream()), name)
    for k in range(m):
        h, w = (int(v) for v in hw[k])
        out["seam"].append(seam[off[k]:off[k + 1]].view(h, w))
        out["blend"].append(blend[off[k]:off[k + 1]].view(h, w))
    return out


def _scaled_seam_masks(frames, M, dst_h, dst_w, finder, a):
    """mosaic_seam_masks at scale a < 1."""
    from . import mosaic
    what = "mosaic_seam_masks"
    frames, Mh, sizes = _frames_and_M(frames, M, what, (3,))
    Ms, _, (Hs, Ws) = mosaic.seam_geometry(Mh, sizes, int(dst_h), int(dst_w), a)
    found = mosaic_seam_masks([resize_linear_exact_u8(f, scale=a) for f in frames], Ms, Hs, Ws, finder)
    fed = _Fed(frames, Mh, dst_h, dst_w, what, _lib.SEAM_MAX_FRAMES)
    out = dict(take=fed.take, rois=fed.rois, seam=[], blend=[], seam_rois=found["rois"], scale=a)
    if "cut" in found:
        out["cut"] = found["cut"]
    if not fed.m:
        return out
    m, dev, rr = fed.m, fed.dev, fed.rr
    seam_rr = np.zeros((m, 4), np.int32)
    seam_ptrs = (ctypes.c_void_p * m)()
    for q, k in enumerate(fed.take):
        if k in found["take"]:
            t = found["seam"][found["take"].index(k)]
            seam_rr[q] = found["rois"][k]
            seam_ptrs[q] = t.data_ptr()
        else:
            t = torch.zeros((0, 0), device=dev, dtype=torch.uint8)
        out["seam"].append(t)
    area = (rr[:, 2] - rr[:, 0]).astype(np.int64) * (rr[:, 3] - rr[:, 1])
    off = np.concatenate([[0], np.cumsum(area)])
    blend = torch.empty(int(off[-1]), device=dev, dtype=torch.uint8)
    nb = lib.udh_mosaic_seam_upscale_workspace_bytes(rr.ctypes.data, seam_rr.ctypes.data, m, Hs, Ws, a, int(dst_h), int(dst_w))
    if nb == 0:
        raise _lib.UdhError("%s: bad arguments (%d frames, canvas %dx%d, seam canvas %dx%d)" % (what, m, dst_h, dst_w, Hs, Ws))
    ws = torch.empty(nb, device=dev, dtype=torch.uint8)
    check(lib.udh_mosaic_seam_upscale_u8(fed.ptrs, fed.sz.ctypes.data, _ptr(fed.M_d), rr.ctypes.data, seam_ptrs, seam_rr.ctypes.data, m,
                                         Hs, Ws, a, int(dst_h), int(dst_w), _ptr(blend), _ptr(ws), nb, _stream()),
          "udh_mosaic_seam_upscale_u8")
    for k in range(m):
        out["blend"].append(blend[off[k]:off[k + 1]].view(int(rr[k, 3] - rr[k, 1]), int(rr[k, 2] - rr[k, 0])))
    return out


def grid_mincut(hcap, vcap, src, snk, residual=False):
    """The minimum cut of an h x w 4-connected grid graph (udh_debug_grid_mincut): hcap, vcap, src, snk CUDA int32
    [h,w] (hcap[y,x]: edge (x, y) - (x + 1, y), both ways; vcap[y,x]: edge (x, y) - (x, y + 1); src / snk: terminal
    capacities; all in [0, 2^24]) -> dict(T CUDA uint8 [h,w]: 1 where the pixel reaches the sink in the residual graph of
    a maximum preflow, cut: the cut's capacity (int), and with residual=True residual CUDA int32 [5,h,w]: the residual
    capacities to the right, lower, left and upper neighbour and to the sink)."""
    for t, nm in ((hcap, "hcap"), (vcap, "vcap"), (src, "src"), (snk, "snk")):
        _req(t, torch.int32, nm)
        if t.dim() != 2 or t.shape != hcap.shape:
            raise _lib.UdhError("grid_mincut: %s must be [h,w] like hcap (got %s)" % (nm, tuple(t.shape)))
    h, w = (int(v) for v in hcap.shape)
    nb = lib.udh_debug_grid_mincut_workspace_bytes(h, w)
    if nb == 0:
        raise _lib.UdhError("grid_mincut: bad dimensions %dx%d" % (h, w))
    dev = hcap.device
    ws = torch.empty(nb, device=dev, dtype=torch.uint8)
    T = torch.empty((h, w), device=dev, dtype=torch.uint8)
    res = torch.empty((5, h, w), device=dev, dtype=torch.int32) if residual else None
    cut = ctypes.c_int64(0)
    check(lib.udh_debug_grid_mincut(_ptr(hcap), _ptr(vcap), _ptr(src), _ptr(snk), h, w, _ptr(T), ctypes.addressof(cut), _ptr(res), _ptr(ws),
                                    nb, _stream()), "udh_debug_grid_mincut")
    out = dict(T=T, cut=int(cut.value))
    if residual:
        out["residual"] = res
    return out


# ------------------------------------------------------------------ Adam
def adam_step(p, g, m, v, alpha_t, beta1=0.9, beta2=0.999, eps=1e-8, grad_scale=1.0, zero_grad=True):
    for t, n in ((p, "p"), (g, "g"), (m, "m"), (v, "v")):
        _req(t, torch.float32, n)
    check(lib.udh_adam_step(_ptr(p), _ptr(g), _ptr(m), _ptr(v), p.numel(), float(alpha_t), float(beta1), float(beta2),
                            float(eps), float(grad_scale), int(bool(zero_grad)), _stream()), "udh_adam_step")
