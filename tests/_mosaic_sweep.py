"""A synthetic camera sweep over one smooth texture, with its true homographies (shared by the mosaic tests and
tools/mosaic_time.py): frame k is the texture seen through A_k (frame pixel -> texture pixel), so the true pair
homography (frame k -> frame k + 1) is inv(A_{k+1}) A_k and frame k -> the reference frame is inv(A_ref) A_k."""
import numpy as np


def texture(rng, h, w):
    """A smooth uint8 RGB texture: bicubic upscale of 1/16-resolution noise (two bilinear resamplings of it differ little)."""
    import cv2
    small = rng.integers(0, 256, (h // 16 + 3, w // 16 + 3, 3)).astype(np.float32)
    return np.clip(cv2.resize(small, (w, h), interpolation=cv2.INTER_CUBIC), 0, 255).astype(np.uint8)


def camera(cx, cy, h, w, angle, scale, px, py):
    """Frame pixel -> texture pixel: the frame's centre at (cx, cy), rotated, scaled, with a perspective term."""
    c, s = np.cos(angle) * scale, np.sin(angle) * scale
    P = np.array([[1.0, 0, 0], [0, 1.0, 0], [px, py, 1.0]])
    A = np.array([[c, -s, cx], [s, c, cy], [0, 0, 1.0]]) @ P @ np.array([[1.0, 0, -(w - 1) / 2.0], [0, 1.0, -(h - 1) / 2.0], [0, 0, 1.0]])
    return A / A[2, 2]


def sweep_cameras(n, h, w, overlap=0.6, seed=0):
    """n cameras panning right with about `overlap` of a frame shared by neighbours -> (A [n,3,3], texture size (th, tw))."""
    rng = np.random.default_rng(seed)
    step = (1.0 - overlap) * w
    margin = 0.15 * max(h, w)
    A = np.stack([camera(margin + (w - 1) / 2.0 + k * step, margin + (h - 1) / 2.0 + rng.uniform(-0.03, 0.03) * h, h, w,
                         rng.uniform(-0.03, 0.03), rng.uniform(0.97, 1.03), rng.uniform(-3e-5, 3e-5) * 320.0 / w,
                         rng.uniform(-3e-5, 3e-5) * 320.0 / w) for k in range(n)])
    return A, (int(h + 2 * margin), int(w + (n - 1) * step + 2 * margin))


def sweep(n, h, w, overlap=0.6, seed=0):
    """-> (texture uint8 [th,tw,3], frames [n] uint8 [h,w,3], A [n,3,3], true pair H [n-1,3,3])."""
    import cv2
    A, (th, tw) = sweep_cameras(n, h, w, overlap, seed)
    tex = texture(np.random.default_rng(seed + 1000), th, tw)
    frames = [cv2.warpPerspective(tex, A[k], (w, h), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP) for k in range(n)]
    return tex, frames, A, true_pairs(A)


def true_pairs(A):
    H = np.stack([np.linalg.inv(A[k + 1]) @ A[k] for k in range(len(A) - 1)])
    return H / H[:, 2:3, 2:3]
