"""Correspondence-based test metric of the real-data path (code/homography_CNN_real.py:578-612), in NumPy.

The aerial test set has no 4-point ground truth; each test line of `test_gt.txt` holds 16 numbers: four hand-picked
correspondences (x,y) in image 1 followed by their matches in image 2, clicked on 480x640 frames (hence the /2 onto the
240x320 "full" images, :599-600).  For a predicted h4p on the network-size image (img_h x img_w = 142x190):
    full_pts1 = pts1 * r,  full_pts2 = (pts1 + h4p) * r,  r = full_img_h / img_h                      (:588-596)
    full_H = getPerspectiveTransform(full_pts1, full_pts2);  pred_corr2 = perspectiveTransform(corr1, inv(full_H))   (:598-604)
    h_loss = RMSE(pred_corr2 - corr2) over the 8 coordinates; identity = RMSE(corr1 - corr2);
    a sample FAILS when h_loss > identity and is then counted with the identity error                        (:607-614)
"""
import numpy as np


def get_perspective_transform(src, dst):
    """cv2.getPerspectiveTransform: src, dst [4,2] -> H [3,3] with h33 = 1 (the same 8x8 system as the reference's DLT)."""
    src, dst = np.asarray(src, np.float64), np.asarray(dst, np.float64)
    A, b = np.zeros((8, 8)), np.zeros(8)
    for i in range(4):
        x, y = src[i]; u, v = dst[i]
        A[i] = [x, y, 1, 0, 0, 0, -x * u, -y * u]; b[i] = u
        A[i + 4] = [0, 0, 0, x, y, 1, -x * v, -y * v]; b[i + 4] = v
    return np.append(np.linalg.solve(A, b), 1.0).reshape(3, 3)


def perspective_transform(pts, H):
    p = np.concatenate([np.asarray(pts, np.float64), np.ones((len(pts), 1))], axis=1) @ np.asarray(H, np.float64).T
    return p[:, :2] / p[:, 2:3]


def correspondence_errors(pred_h4p, pts1, gt_corr, full_img_h=240, img_h=142, corr_scale=0.5, with_points=False):
    """Per-sample (h_loss, identity_loss, failed) as the reference's test loop computes them.  pred_h4p, pts1: [B,8];
    gt_corr: [B,16] = corr1 (4 x (x,y)) then corr2, in the frame the points were clicked on (corr_scale maps it onto the
    full images: 1/2 in the reference).  with_points: each tuple also carries pred_corr2 [4,2] (float64), the predicted
    matches of corr1 that the report image draws."""
    r = float(full_img_h) / float(img_h)
    out = []
    for h4p, p1, gc in zip(np.asarray(pred_h4p, np.float64), np.asarray(pts1, np.float64), np.asarray(gt_corr, np.float64)):
        full_pts1 = p1.reshape(4, 2) * r
        full_pts2 = (h4p.reshape(4, 2) + p1.reshape(4, 2)) * r
        H = get_perspective_transform(full_pts1.astype(np.float32), full_pts2.astype(np.float32))
        corr1, corr2 = gc[:8].reshape(4, 2) * corr_scale, gc[8:16].reshape(4, 2) * corr_scale
        pred_corr2 = perspective_transform(corr1, np.linalg.inv(H))
        h_loss = float(np.sqrt(np.mean(np.square(pred_corr2 - corr2))))
        ident = float(np.sqrt(np.mean(np.square(corr1 - corr2))))
        failed = h_loss > ident
        res = (ident if failed else h_loss, ident, bool(failed))
        out.append(res + (pred_corr2,) if with_points else res)
    return out
