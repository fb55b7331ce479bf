"""Batched mirror of code/utils/direct_homography.py: the direct (ECC) homography baseline on the device.

find_homography(img1, img2, H4p1) takes a batch where the reference takes one pair: uint8 gray planes [B,H,W] (the
reference converts its RGB inputs with cvtColor RGB2GRAY first; ops.ecc_prep_u8 produces exactly the planes the
conventional harness hands over) and the patch corners H4p1 [B,8].  Per sample it runs
cv2.findTransformECC(img1, img2, I, MOTION_HOMOGRAPHY, (COUNT|EPS, num_iterations, 1e-10)) in libudh's CUDA kernel and
returns (pred_h4p [B,8], W [B,3,3], not_found [B] bool): the reference's (transformedCorners - corners, M, 1 on
exception), with pred_h4p = 0 where ECC raised.  The harness's clamp to +-2 rho is applied only when rho is given.
"""
import torch

from . import _lib, ops

_NO_CLAMP = 3.0e38


def find_homography(img1, img2, H4p1, num_iterations=100, rho=None, eps=1e-10):
    for t, n in ((img1, "img1"), (img2, "img2")):
        if not (isinstance(t, torch.Tensor) and t.is_cuda):
            raise _lib.UdhError("%s must be a CUDA tensor (libudh has no CPU path)" % n)
        if t.dim() != 3 or t.dtype != torch.uint8:
            raise _lib.UdhError("%s must be uint8 gray planes [B,H,W] (see ops.ecc_prep_u8 for RGB inputs)" % n)
    W, _, _, status = ops.find_homography_ecc(img1.contiguous(), img2.contiguous(), None, num_iterations, eps)
    pts = H4p1.reshape(-1, 8).to(device=img1.device, dtype=torch.float32).contiguous()
    pred, _, _ = ops.ecc_h4p(W, status, pts, None, _NO_CLAMP if rho is None else float(rho))
    return pred, W, status != _lib.ECC_OK
