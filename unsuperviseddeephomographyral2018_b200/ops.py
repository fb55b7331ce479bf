"""Torch-tensor wrappers over the C ABI (include/udh.h).  PyTorch is plumbing here: device memory, streams and
autograd bookkeeping; all arithmetic happens in libudh's CUDA kernels.  Every function requires CUDA tensors."""
import ctypes

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
    nbytes = lib.udh_ecc_workspace_bytes(B, Hh, W)
    ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    check(lib.udh_ecc_homography(_ptr(template), _ptr(image), _ptr(W_init), int(max_iters), float(eps), _ptr(Wout), _ptr(rho),
                                 _ptr(iters), _ptr(status), _ptr(ws), nbytes, B, Hh, W, _stream()), "udh_ecc_homography")
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


# ------------------------------------------------------------------ Adam
def adam_step(p, g, m, v, alpha_t, beta1=0.9, beta2=0.999, eps=1e-8, grad_scale=1.0, zero_grad=True):
    for t, n in ((p, "p"), (g, "g"), (m, "m"), (v, "v")):
        _req(t, torch.float32, n)
    check(lib.udh_adam_step(_ptr(p), _ptr(g), _ptr(m), _ptr(v), p.numel(), float(alpha_t), float(beta1), float(beta2),
                            float(eps), float(grad_scale), int(bool(zero_grad)), _stream()), "udh_adam_step")
