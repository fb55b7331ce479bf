"""Report images of the test harnesses (--save_visual): the reference's save_correspondences_img (utils/utils.py:209-307)
for a whole batch in one launch.

The two images side by side, the prediction polygon on the right one, the ground-truth polygons and the four matches
drawn over them, written as JPEG files byte-identical to cv2.imwrite's.  The integer conversions of the points stay here,
with NumPy's own semantics (astype truncation, np.round half to even, np.int32(nan) = INT_MIN); the device only
rasterises (ops.draw_report_u8) and encodes (ops.encode_jpeg, quality 95).  One deliberate difference: draw_matches also
writes every canvas to a scratch file (/tmp/tmp.jpg) that nothing reads; that file is not written.
"""
import os

import numpy as np
import torch

from . import ops


def report_vertices(corr1, corr2, pred_corr2, w1):
    """Points of one sample [4,2] -> the int32 vertices [20,2] the reference hands cv2: the prediction polygon
    np.int32(pred_corr2) (right-image coordinates), kp2 = (corr2 + [w1, 0]).astype(int32), kp1 = corr1.astype(int32),
    the match lines' starts np.round(kp1) and ends np.round(corr2) + [w1, 0] (from the float corr2)."""
    corr1, corr2, pred = np.asarray(corr1), np.asarray(corr2), np.asarray(pred_corr2)
    with np.errstate(invalid="ignore"):
        pred_i = np.int32(pred)
        kp2 = (corr2 + np.array([w1, 0])).astype(np.int32)
    kp1 = corr1.astype(np.int32)
    end1 = np.round(kp1).astype(int)
    end2 = np.round(corr2).astype(int) + np.array([w1, 0])
    if np.abs(end2).max() >= 2 ** 31:
        raise ValueError("report_vertices: a match end point is outside int32 (cv2.line rejects it)")
    return np.concatenate([pred_i, kp2, kp1, end1, end2.astype(np.int32)]).reshape(20, 2).astype(np.int32)


def render(batch, idx, corr1, corr2, pred_corr2, prime_left):
    """Canvases [n,h,2w,3] uint8 (CUDA) of the batch's samples idx: I_u8 / I_prime_u8 / aug of the loader batch, the
    points [n,4,2] per sample; prime_left puts I' on the left (the synthetic harness) instead of I."""
    idx = torch.as_tensor(np.asarray(idx, np.int64), device=batch["I_u8"].device)
    I, Ip = batch["I_u8"].index_select(0, idx).contiguous(), batch["I_prime_u8"].index_select(0, idx).contiguous()
    aug = batch.get("aug")
    aug = aug.index_select(0, idx).contiguous() if aug is not None else None
    w = I.shape[2]
    verts = np.stack([report_vertices(a, b, c, w) for a, b, c in zip(corr1, corr2, pred_corr2)])
    return ops.draw_report_u8(I, Ip, aug, torch.from_numpy(verts).to(I.device), prime_left)


def write(canvases, names, results_dir):
    """Encode the canvases (cv2.imwrite's JPEG, quality 95) and write them as results_dir/name."""
    os.makedirs(results_dir, exist_ok=True)
    for name, blob in zip(names, ops.encode_jpeg(canvases, quality=95)):
        path = os.path.join(results_dir, name)
        with open(path, "wb") as f:
            f.write(blob)
        print('Wrote file %s', path)


def synthetic_name(step, batch_size, loss_type, h_loss):
    """homography_CNN_synthetic.py:551, with the batch's h_loss as the float32 the session returns."""
    return str(step * batch_size) + '_' + loss_type + '_loss_' + str(np.float32(h_loss)) + '.jpg'


def synthetic_points(pts1, gt, pred_h4p):
    """Sample points of the synthetic harness (:542-548): corr1 = pts1, corr2 = pts1 + gt, pred = pts1 + pred_h4p, all
    float32 [n,4,2]."""
    p1 = np.asarray(pts1, np.float32).reshape(-1, 4, 2)
    return p1, p1 + np.asarray(gt, np.float32).reshape(-1, 4, 2), p1 + np.asarray(pred_h4p, np.float32).reshape(-1, 4, 2)


def global_index(rank, per_gpu, step, batch_size, i):
    """The reference's image index k = step*batch_size + i (homography_CNN_real.py:616), made global over the ranks:
    rank r's sample i of a step is sample r*per_gpu + i of the global batch."""
    return rank * per_gpu + step * batch_size + i


def real_cnn_name(k, h_loss):
    """homography_CNN_real.py:616, h_loss after the failure substitution."""
    return str(k) + '_Unsupervised_' + '_loss_' + str(h_loss) + '.jpg'


def conventional_name(k, h_loss):
    """homography_conventional_real.py:263."""
    return str(k) + '_loss_' + str(h_loss) + '.jpg'


def clicked_points(gt_corr):
    """corr1, corr2 [n,4,2] of the real harnesses: the clicked correspondences [n,16] halved onto the full-size images
    (float32, as the session returns them)."""
    g = np.asarray(gt_corr, np.float32).reshape(-1, 16)
    return g[:, 0:8].reshape(-1, 4, 2) / 2, g[:, 8:16].reshape(-1, 4, 2) / 2
