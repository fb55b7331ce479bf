"""Synthetic pairs for the refinement tests: a multi-octave value-noise RGB texture (detail at every pyramid level),
image 2 = cv2.warpPerspective(image 1, H_true), and a starting H whose corners are off by up to `perturb` px in the
240x320 network frame."""
import cv2
import numpy as np


def texture(h, w, seed):
    """uint8 RGB [h,w,3]: bicubic value noise with cells of 4, 8, ... px up to a quarter of the short side."""
    rng = np.random.default_rng(seed)
    img = np.zeros((h, w, 3), np.float32)
    cell = 4
    while cell <= min(h, w) // 4:
        g = rng.random((h // cell + 2, w // cell + 2, 3)).astype(np.float32)
        img += cv2.resize(g, (w + 2 * cell, h + 2 * cell), interpolation=cv2.INTER_CUBIC)[cell:cell + h, cell:cell + w]
        cell *= 2
    img -= img.min()
    return np.clip(img * (255.0 / img.max()), 0, 255).astype(np.uint8)


def corners(h, w):
    return np.array([[0, 0], [w - 1, 0], [w - 1, h - 1], [0, h - 1]], np.float64)


def apply(H, pts):
    p = np.c_[pts, np.ones(len(pts))] @ np.asarray(H, np.float64).reshape(3, 3).T
    return p[:, :2] / p[:, 2:]


def corner_error(Ha, Hb, h, w):
    """Largest distance between where Ha and Hb send image 1's corners (px)."""
    return float(np.abs(apply(Ha, corners(h, w)) - apply(Hb, corners(h, w))).max())


def true_homography(h, w, seed):
    """A mild homography about the image centre: rotation up to 3 degrees, scale 0.97..1.03, shift up to 3 % of the size,
    perspective up to 1e-5 per px at 480x640."""
    rng = np.random.default_rng(seed + 1000)
    a = np.deg2rad(rng.uniform(-3, 3)); s = rng.uniform(0.97, 1.03)
    c = np.array([[1, 0, (w - 1) / 2.0], [0, 1, (h - 1) / 2.0], [0, 0, 1]])
    R = np.array([[s * np.cos(a), -s * np.sin(a), rng.uniform(-0.03, 0.03) * w],
                  [s * np.sin(a), s * np.cos(a), rng.uniform(-0.03, 0.03) * h],
                  [rng.uniform(-1e-5, 1e-5) * 640.0 / w, rng.uniform(-1e-5, 1e-5) * 480.0 / h, 1]])
    H = c @ R @ np.linalg.inv(c)
    return H / H[2, 2]


def pair(h, w, seed, perturb):
    """-> (img1, img2, H_true, H_start): image 2 = warpPerspective(image 1, H_true); H_start sends image 1's corners up to
    `perturb` px (in the 240x320 frame, i.e. perturb * h / 240 px here) away from H_true's."""
    img1 = texture(h, w, seed)
    Ht = true_homography(h, w, seed)
    img2 = cv2.warpPerspective(img1, Ht, (w, h))
    rng = np.random.default_rng(seed + 2000)
    c = corners(h, w).astype(np.float32)
    d = rng.uniform(-1, 1, (4, 2)) * perturb * (h / 240.0)
    H0 = cv2.getPerspectiveTransform(c, (apply(Ht, c) + d).astype(np.float32))
    return img1, img2, Ht, H0 / H0[2, 2]
