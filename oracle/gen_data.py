"""Host restatement of the dataset generator's pixel work (test reference and timing baseline, not a CLI option).

warp(img, theta)    numpy_spatial_transformer._transform / _interpolate as the generator calls them, per channel (the
                    reference's 3-D branch relies on an old-NumPy expand_dims leniency): np.linspace grid, np.dot,
                    x / t, (x + 1) * W / 2, floor, clip, weights from the clipped corners, wa Ia + wb Ib + wc Ic + wd Id,
                    astype(uint8).
gray(bgr)           cv2.cvtColor(bgr, COLOR_RGB2GRAY) as the generator calls it on a BGR image.
HostBackend         cv2.resize + gray + warp + cv2.imencode: unsuperviseddeephomographyral2018_b200.gen_data.generate
                    with it is the host generator the device generator is compared with.
reference_draws     a transcription of homographyGeneration / dataCollection's loop (draws, indices, cutoffs).
"""
import random

import numpy as np


def warp(img, theta):
    """uint8 [h,w] or [h,w,C], theta [3,3] float64 -> uint8 of the same shape."""
    h, w = img.shape[:2]
    x_t, y_t = np.meshgrid(np.linspace(-1, 1, w), np.linspace(-1, 1, h))
    grid = np.vstack([x_t.flatten(), y_t.flatten(), np.ones(np.prod(x_t.shape))])
    T = np.dot(np.reshape(theta, (3, 3)), grid)
    x = np.reshape(T[0, :], [-1]) / np.reshape(T[2, :], [-1])
    y = np.reshape(T[1, :], [-1]) / np.reshape(T[2, :], [-1])
    x = (x + 1.0) * float(w) / 2.0
    y = (y + 1.0) * float(h) / 2.0
    x0 = np.floor(x).astype(int)
    x1 = x0 + 1
    y0 = np.floor(y).astype(int)
    y1 = y0 + 1
    zero = np.zeros([], dtype="int32")
    x0, x1 = np.clip(x0, zero, w - 1), np.clip(x1, zero, w - 1)
    y0, y1 = np.clip(y0, zero, h - 1), np.clip(y1, zero, h - 1)
    wa = (x1 - x) * (y1 - y)
    wb = (x1 - x) * (y - y0)
    wc = (x - x0) * (y1 - y)
    wd = (x - x0) * (y - y0)

    def one(im):
        out = wa * im[y0, x0] + wb * im[y1, x0] + wc * im[y0, x1] + wd * im[y1, x1]
        with np.errstate(invalid="ignore"):
            return np.reshape(out, [h, w]).astype(np.uint8)

    if img.ndim == 2:
        return one(img)
    return np.stack([one(img[..., c]) for c in range(img.shape[2])], axis=2)


def gray(bgr):
    """cv2.cvtColor(bgr, COLOR_RGB2GRAY): 15-bit fixed point, round half up, channel 0 weighted as R."""
    c = bgr.astype(np.int64)
    return ((c[..., 0] * 9798 + c[..., 1] * 19235 + c[..., 2] * 3735 + 16384) >> 15).astype(np.uint8)


class HostBackend:
    """cv2.resize, gray, warp and cv2.imencode (cv2.imwrite's bytes) on the host."""

    def __init__(self, quality=95):
        self.quality = quality

    def pairs(self, raws, which, thetas, height, width, gray_files):
        import cv2
        enc = lambda im: cv2.imencode(".jpg", im, [cv2.IMWRITE_JPEG_QUALITY, self.quality])[1].tobytes()
        resized = [cv2.resize(r, (width, height)) for r in raws]
        out_i, out_p = [], []
        for k, th in zip(which, thetas):
            c = resized[k]
            g = gray(c)
            if gray_files:
                out_i.append(enc(g)); out_p.append(enc(warp(g, th)))
            else:
                out_i.append(enc(c)); out_p.append(enc(warp(c, th)))
        return out_i, out_p


def reference_draws(readable, num_data, start_index, img_per_real, rho=45, patch_size=128, height=240, width=320, seed=0):
    """homographyGeneration's loop over the raw list, transcribed: readable[k] says whether raw image k loads.
    -> [(index, four_points, perturbed_four_points)] of the pairs written."""
    rnd = random.Random(seed)
    out, index = [], start_index
    for ok in readable:
        if not ok:
            continue
        for i in range(img_per_real):
            y = rnd.randint(rho, height - rho - patch_size)
            x = rnd.randint(rho, width - rho - patch_size)
            top_left_point = (x, y)
            bottom_left_point = (patch_size + x, y)
            bottom_right_point = (patch_size + x, patch_size + y)
            top_right_point = (x, patch_size + y)
            four_points = [top_left_point, bottom_left_point, bottom_right_point, top_right_point]
            perturbed_four_points = []
            for point in four_points:
                perturbed_four_points.append((point[0] + rnd.randint(-rho, rho), point[1] + rnd.randint(-rho, rho)))
            out.append((index, four_points, perturbed_four_points))
            index += 1
            if index >= num_data + start_index:
                break
        if index >= num_data + start_index:
            break
    return out
