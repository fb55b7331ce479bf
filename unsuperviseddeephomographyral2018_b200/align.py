"""Align any two images with a trained model: the homography between image 1 and image 2 in their own pixels, and image 1
warped into image 2's frame.

    est = HomographyEstimator(model_prefix=None, engine=None, img_h=240, img_w=320, patch_size=128, numeric="bf16x3",
                              batch_size=128)
    H, pred_h4p, pts1 = est.estimate(I1_u8, I2_u8, corners=None)
    warped = est.warp(I1_u8, H, (H2, W2))

Images are CUDA uint8 RGB (the real-data loader's channel order), either one [B,h,w,3] tensor per side or a list of
[h,w,3] tensors of any sizes.  The defaults describe the synthetic model; img_h=142, img_w=190 describe the real-data one.

Preprocessing is the real-data loader's in test mode without augmentation, each image taken as its own full-size image:
RGB values through the loader's normalise table (synthetic.MEAN_I / STD_I), then to img_h x img_w by
  * "device"          udh_real_prep: the table and, when the sizes differ, cv2's generic INTER_AREA downscale;
  * "device-upscale"  an image smaller on both axes: cv2's uint8 INTER_AREA upscale (udh_resize_area_up_u8, the loader's
                      rule for files below the full size), then the table;
  * "host"            every other size (ops.area_is_generic is False: integer ratios, one axis up): the loader's host
                      fallback, cv2.resize(INTER_AREA) of the normalised fp32 image, one image at a time.
Camera frames take the device path: udh_real_prep reads the source rows of an output row from global memory when they do
not fit in shared memory (3000 x 4000 -> 240 x 320 sums 14 rows of 4000 px per output row), with the same sums.
`prep_paths` maps each image size of the last estimate() to the path it took.  The patch is the centred patch_size square
of the network frame unless `corners` ([B,8], network frame, the loader's pts1 layout: an axis-aligned patch_size square
with integer corners inside the frame, checked) gives it; patch_indices and the
gray patches are the loader's.  The forward is engine.forward(batch, train=False); a short last batch is padded with
copies of its first pair, and no pair's result depends on the others (each item of the network is computed alone).

Convention.  The network predicts pred_h4p, the displacements that take the patch corners pts1 of image 2 to their
matches in image 1, on img_h x img_w images.  With S_k = diag(w_k / img_w, h_k / img_h, 1) the scale from the network
frame to image k (h_k x w_k), the real-data test metric's rule (real_metrics.correspondence_errors) becomes
    G = getPerspectiveTransform(float32(S_2 pts1), float32(S_1 (pts1 + pred_h4p)))       (image 2 -> image 1)
    H = inv(G) / inv(G)[2,2]                                                             (image 1 -> image 2)
so that x2 ~ H x1 in original pixels, and cv2.warpPerspective(I1, H, (w2, h2)) lays image 1 over image 2.  When both
images have the metric's full size and the resize keeps the aspect ratio (S_1 = S_2 = r I), H x1 is the metric's
pred_corr2; the metric scales both axes by full_img_h / img_h, which differs from S_k where the aspect ratio changes
(240 x 320 -> 142 x 190 by 0.35 % in x).

Refinement.  est.refine(I1, I2, H, levels, iters, eps, max_side) improves H on the images' own pixels with coarse-to-fine
ECC (cv2.findTransformECC, MOTION_HOMOGRAPHY, on the split-pair kernel udh_ecc_homography_split):
  * levels     refine_level_sizes: the finest level is image 2's size, or that size scaled to a long side of max_side;
               each coarser level is ((h + 1) // 2, (w + 1) // 2), and levels whose short side would fall below
               MIN_LEVEL_SIDE are not made.  levels=None (the default) halves until the long side is at most 320 px,
               about the network frame the estimate came from.  Both images of a pair are resized to the level's size;
  * planes     cvtColor(cv2.resize(img, (w_k, h_k)), RGB2GRAY) (ops.resize_linear_u8, ops.gray_u8; no resize at the
               image's own size);
  * coordinates  cv2.resize's pixel-centre map x_k = (x + 0.5) s - 0.5 per axis (level_transform), so
               W_k = inv(T2k H T1k^-1) (template: image 2's plane, input: image 1's; to_level) and back
               H = T2k^-1 inv(W_k) T1k (from_level), all in float64 with W_k rounded to float32 as cv2 takes it;
  * per level  findTransformECC(template, input, W_k, MOTION_HOMOGRAPHY, (COUNT | EPS, iters, eps), None, 5);
  * failures   a pair whose level ends with a non-zero status (where cv2 raises) keeps the H it had before that level
               and runs no finer level; status is that level's, level_reached counts the levels that succeeded.
oracle/ecc_refine.py restates the schedule with cv2 calls.
"""
import collections
import math
import os

import numpy as np
import torch

from . import dataloader as dl, ops, real_metrics as rm

PREP_DEVICE, PREP_DEVICE_UPSCALE, PREP_HOST = "device", "device-upscale", "host"


def image_homography(pred_h4p, pts1, size1, size2, img_h, img_w):
    """pred_h4p, pts1 [B,8] (network frame), size1 / size2 = (h, w) of image 1 / image 2 -> H float64 [B,3,3], H[2,2] = 1,
    x2 ~ H x1 in original pixels (the module docstring's convention)."""
    h4p = np.asarray(pred_h4p, np.float64).reshape(-1, 4, 2)
    p1 = np.asarray(pts1, np.float64).reshape(-1, 4, 2)
    s1 = np.array([size1[1] / float(img_w), size1[0] / float(img_h)])
    s2 = np.array([size2[1] / float(img_w), size2[0] / float(img_h)])
    out = np.empty((len(h4p), 3, 3))
    for k in range(len(h4p)):
        G = rm.get_perspective_transform((p1[k] * s2).astype(np.float32), ((h4p[k] + p1[k]) * s1).astype(np.float32))
        H = np.linalg.inv(G)
        out[k] = H / H[2, 2]
    return out


def centred_corners(n, img_h, img_w, patch_size):
    """[n,8] float32: the centred patch_size square of the network frame in the loader's pts1 layout."""
    x0, y0 = (img_w - patch_size) // 2, (img_h - patch_size) // 2
    P = patch_size
    return np.tile(np.array([x0, y0, x0 + P, y0, x0 + P, y0 + P, x0, y0 + P], np.float32), (n, 1))


def prep_path(h, w, img_h, img_w):
    """The path an h x w image takes to the network size (the module docstring's three)."""
    if (h, w) == (img_h, img_w):
        return PREP_DEVICE
    if ops.area_is_generic(h, w, img_h, img_w):
        return PREP_DEVICE
    if h < img_h and w < img_w:
        return PREP_DEVICE_UPSCALE
    return PREP_HOST


def check_corners(corners, n, img_h, img_w, patch_size):
    """corners [n,8] (network frame) -> float32 [n,8], or ValueError unless every row is the loader's pts1 of an
    axis-aligned patch_size square with integer corners inside img_h x img_w: the patch is gathered from the first corner
    and all eight go to the DLT, so anything else would index outside the image or disagree with the patch."""
    c = np.asarray(corners, np.float64)
    if c.size != 8 * n:
        raise ValueError("corners must be [%d,8] (got %d values)" % (n, c.size))
    c = c.reshape(n, 8)
    x0, y0, P = c[:, 0:1], c[:, 1:2], patch_size
    square = np.concatenate([x0, y0, x0 + P, y0, x0 + P, y0 + P, x0, y0 + P], 1)
    bad = ~(np.isfinite(c).all(1) & (c == np.round(c)).all(1) & (c == square).all(1) & (x0[:, 0] >= 0) & (y0[:, 0] >= 0)
            & (x0[:, 0] + P <= img_w) & (y0[:, 0] + P <= img_h))
    if bad.any():
        k = int(np.flatnonzero(bad)[0])
        raise ValueError("corners[%d] = %s is not an integer %dx%d square inside the %dx%d network frame"
                         % (k, c[k].tolist(), P, P, img_h, img_w))
    return c.astype(np.float32)


# ---- refinement schedule (the module docstring's "Refinement") --------------------------------------------------------
MIN_LEVEL_SIDE = 16
# levels=None: halve until the long side is at most AUTO_COARSEST_SIDE, about the network frame the estimate came from
# (its error there is a few px); coarser levels can lose what the estimate had on textures with little coarse detail
AUTO_COARSEST_SIDE = 320
REFINE_LEVELS, REFINE_ITERS, REFINE_EPS = None, 50, 1e-6
REFINE_PIXELS = 1 << 28          # pixels of the finest level per split-kernel batch (2 GB of workspace)


def refine_level_sizes(h, w, levels=None, max_side=None):
    """[(h_k, w_k)] coarsest first, for image 2 of size h x w: the finest h x w or scaled to a long side of max_side
    (rounded half up), each coarser one ((h + 1) // 2, (w + 1) // 2), none with a short side below MIN_LEVEL_SIDE except
    the finest; at most `levels` levels, or with levels=None until the long side is at most AUTO_COARSEST_SIDE."""
    if levels is not None and levels < 1:
        raise ValueError("levels must be >= 1 (got %d)" % levels)
    if max_side is not None:
        if max_side < 2:
            raise ValueError("max_side must be >= 2 (got %d)" % max_side)
        if max(h, w) > max_side:
            s = max_side / float(max(h, w))
            h, w = max(1, int(math.floor(h * s + 0.5))), max(1, int(math.floor(w * s + 0.5)))
    if min(h, w) < 2:
        raise ValueError("the finest level %dx%d is smaller than 2x2" % (h, w))
    sizes = [(h, w)]
    while len(sizes) < levels if levels is not None else max(h, w) > AUTO_COARSEST_SIDE:
        h, w = (h + 1) // 2, (w + 1) // 2
        if min(h, w) < MIN_LEVEL_SIDE:
            break
        sizes.append((h, w))
    return sizes[::-1]


def level_transform(size, size_k):
    """3x3 float64 taking pixel coordinates of an image of size (h, w) to those of its cv2.resize to size_k = (h_k, w_k):
    x_k = (x + 0.5) w_k / w - 0.5, y_k likewise."""
    sx, sy = size_k[1] / float(size[1]), size_k[0] / float(size[0])
    return np.array([[sx, 0.0, 0.5 * sx - 0.5], [0.0, sy, 0.5 * sy - 0.5], [0.0, 0.0, 1.0]])


def to_level(H, size1, size2, size_k):
    """H [n,3,3] (image 1 -> image 2, original pixels) -> ECC's W_k float32 [n,3,3] at level size_k: inv(T2k H T1k^-1),
    normalised to W_k[2,2] = 1 (template: image 2's plane, input: image 1's)."""
    T1, T2 = level_transform(size1, size_k), level_transform(size2, size_k)
    W = np.linalg.inv(T2 @ np.asarray(H, np.float64).reshape(-1, 3, 3) @ np.linalg.inv(T1))
    return (W / W[:, 2:3, 2:3]).astype(np.float32)


def from_level(W, size1, size2, size_k):
    """ECC's W_k [n,3,3] at level size_k -> H float64 [n,3,3] = T2k^-1 inv(W_k) T1k, normalised to H[2,2] = 1."""
    T1, T2 = level_transform(size1, size_k), level_transform(size2, size_k)
    H = np.linalg.inv(T2) @ np.linalg.inv(np.asarray(W, np.float32).astype(np.float64).reshape(-1, 3, 3)) @ T1
    return H / H[:, 2:3, 2:3]


def _level_plane(I, size_k):
    """uint8 RGB [n,h,w,3] CUDA -> the level's gray planes [n,h_k,w_k]."""
    if tuple(I.shape[1:3]) != tuple(size_k):
        I = ops.resize_linear_u8(I.contiguous(), size_k[0], size_k[1])
    return ops.gray_u8(I.contiguous())


def _as_list(I):
    if isinstance(I, torch.Tensor):
        if I.dim() != 4 or I.shape[3] != 3:
            raise ValueError("images must be [B,h,w,3] uint8 (got %s)" % (tuple(I.shape),))
        return list(I.unbind(0))
    return list(I)


class HomographyEstimator(object):
    def __init__(self, model_prefix=None, engine=None, img_h=240, img_w=320, patch_size=128, numeric="bf16x3", batch_size=128,
                 seed=0):
        """model_prefix: a TF checkpoint prefix (engine.load_tf_checkpoint), or engine: an existing HomographyEngine (its
        batch size, patch and image size are used).  Neither: the engine's seeded initial weights."""
        if engine is None:
            from .engine import HomographyEngine
            engine = HomographyEngine(batch_size, patch_size, img_h, img_w, numeric=numeric, seed=seed)
            if model_prefix is not None:
                engine.load_tf_checkpoint(model_prefix)
        elif model_prefix is not None:
            raise ValueError("give model_prefix or engine, not both")
        self.engine = engine
        self.img_h, self.img_w, self.P, self.B = engine.img_h, engine.img_w, engine.Pz, engine.B
        if self.P > min(self.img_h, self.img_w):
            raise ValueError("patch_size %d does not fit the %dx%d network frame" % (self.P, self.img_h, self.img_w))
        self.prep_paths = {}
        self.last_ms = {}
        self._luts = {}

    # ---- preprocessing ----------------------------------------------------------------------------------------------
    def _plain_luts(self, n):
        if n not in self._luts:
            t = np.ascontiguousarray(np.broadcast_to(dl._value_table(), (n, 4, 256, 3)))
            self._luts[n] = torch.from_numpy(t).to(self.engine.device)
        return self._luts[n]

    def _planes(self, I):
        """uint8 [n,h,w,3] CUDA -> the normalised network-size planes [n,img_h,img_w,3] fp32, by the image size's path."""
        n, h, w, _ = I.shape
        Hh, W = self.img_h, self.img_w
        path = prep_path(h, w, Hh, W)
        self.prep_paths[(h, w)] = path
        if path == PREP_HOST:
            out = [dl.normalise_resize_host(I[j].cpu().numpy().astype(np.float32), Hh, W) for j in range(n)]
            return torch.from_numpy(np.stack(out)).to(I.device)
        if path == PREP_DEVICE_UPSCALE:
            I = ops.resize_area_up_u8(I.contiguous(), Hh, W)
        return ops.real_prep(I.contiguous(), I.contiguous(), self._plain_luts(n), Hh, W)[0]

    def prepare(self, I1, I2, corners=None):
        """One size group: uint8 I1 [n,h1,w1,3], I2 [n,h2,w2,3] (CUDA, RGB) -> the loader's test batch dict (I1, I2,
        I1_aug, I2_aug, I_aug, I_prime_aug, pts1, gt = None, patch_indices) for n pairs."""
        n = I1.shape[0]
        if tuple(I1.shape[1:3]) == tuple(I2.shape[1:3]) and prep_path(I1.shape[1], I1.shape[2], self.img_h, self.img_w) == PREP_DEVICE:
            # the loader's own call: both images of the pair through one udh_real_prep launch
            self.prep_paths[tuple(I1.shape[1:3])] = PREP_DEVICE
            I_pl, Ip_pl = ops.real_prep(I1.contiguous(), I2.contiguous(), self._plain_luts(n), self.img_h, self.img_w)[:2]
        else:
            I_pl, Ip_pl = self._planes(I1), self._planes(I2)
        c = centred_corners(n, self.img_h, self.img_w, self.P) if corners is None else check_corners(corners, n, self.img_h, self.img_w, self.P)
        pts1 = torch.tensor(c, dtype=torch.float32, device=I1.device)
        return dl.gather_patches(I_pl, Ip_pl, I_pl, Ip_pl, pts1, self.P, self.img_w)

    # ---- estimate / warp --------------------------------------------------------------------------------------------
    def _forward(self, batch, n):
        """pred_h4p [n,8] of the first n pairs of a prepared batch, padded to the engine's batch with its first pair."""
        if n < self.B:
            pad = torch.cat([torch.arange(n), torch.zeros(self.B - n, dtype=torch.long)]).to(batch["pts1"].device)
            batch = {k: (v.index_select(0, pad).contiguous() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}
        return self.engine.forward(batch, train=False)["pred_h4p"][:n]

    def estimate(self, I1, I2, corners=None):
        """-> (H float64 [B,3,3], pred_h4p float32 [B,8], pts1 float32 [B,8]) as numpy arrays, pair order kept.  Pairs are
        grouped by (size1, size2); each group runs in engine-sized batches.  last_ms holds the CUDA-event time of the
        prep and forward phases."""
        L1, L2 = _as_list(I1), _as_list(I2)
        if len(L1) != len(L2):
            raise ValueError("%d images 1 for %d images 2" % (len(L1), len(L2)))
        n = len(L1)
        c_all = None if corners is None else check_corners(corners, n, self.img_h, self.img_w, self.P)
        groups = collections.OrderedDict()
        for k in range(n):
            groups.setdefault((tuple(L1[k].shape[:2]), tuple(L2[k].shape[:2])), []).append(k)
        H = np.empty((n, 3, 3)); h4p = np.empty((n, 8), np.float32); pts = np.empty((n, 8), np.float32)
        self.prep_paths = {}
        ev = lambda: torch.cuda.Event(enable_timing=True)
        spans = []
        for (s1, s2), idx in groups.items():
            for c0 in range(0, len(idx), self.B):
                chunk = idx[c0:c0 + self.B]
                e0, e1, e2 = ev(), ev(), ev()
                e0.record()
                batch = self.prepare(torch.stack([L1[k] for k in chunk]), torch.stack([L2[k] for k in chunk]),
                                     None if c_all is None else c_all[chunk])
                e1.record()
                h = self._forward(batch, len(chunk))
                e2.record()
                spans.append((e0, e1, e2))
                h4p[chunk] = h.cpu().numpy()
                pts[chunk] = batch["pts1"][:len(chunk)].cpu().numpy()
            H[idx] = image_homography(h4p[idx], pts[idx], s1, s2, self.img_h, self.img_w)
        torch.cuda.synchronize()
        self.last_ms = dict(prep=sum(a.elapsed_time(b) for a, b, _ in spans), forward=sum(b.elapsed_time(c) for _, b, c in spans))
        return H, h4p, pts

    def warp(self, I1, H, size2):
        """Image 1 warped into image 2's frame: uint8 [B,h1,w1,C] CUDA, H [B,3,3] (image 1 -> image 2), size2 = (h2, w2)
        -> uint8 [B,h2,w2,C], cv2.warpPerspective(I1[b], H[b], (w2, h2)) bit for bit.  last_ms['warp'] is its CUDA-event
        time."""
        M = torch.as_tensor(np.asarray(H, np.float64).reshape(-1, 3, 3)).to(I1.device)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = ops.warp_perspective_u8(I1.contiguous(), M, int(size2[0]), int(size2[1]))
        e1.record()
        e1.synchronize()
        self.last_ms["warp"] = e0.elapsed_time(e1)
        return out

    def refine(self, I1, I2, H, levels=REFINE_LEVELS, iters=REFINE_ITERS, eps=REFINE_EPS, max_side=None):
        """Coarse-to-fine ECC from H (the module docstring's "Refinement").  I1, I2 as for estimate, H [B,3,3] (image 1 ->
        image 2, original pixels) -> (H float64 [B,3,3] with H[2,2] = 1, rho float64 [B] (the last level run; NaN before
        any), status int32 [B] (_lib.ECC_*), level_reached int32 [B]) as numpy arrays.  Pairs are grouped by
        (size1, size2); the host reads each level's result before the next.  last_ms['refine'] is its CUDA-event time."""
        L1, L2 = _as_list(I1), _as_list(I2)
        if len(L1) != len(L2):
            raise ValueError("%d images 1 for %d images 2" % (len(L1), len(L2)))
        n = len(L1)
        H = np.array(H, np.float64).reshape(n, 3, 3)
        H = H / H[:, 2:3, 2:3]
        rho = np.full(n, np.nan); status = np.zeros(n, np.int32); reached = np.zeros(n, np.int32)
        groups = collections.OrderedDict()
        for k in range(n):
            groups.setdefault((tuple(L1[k].shape[:2]), tuple(L2[k].shape[:2])), []).append(k)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for (s1, s2), idx in groups.items():
            sizes = refine_level_sizes(s2[0], s2[1], levels, max_side)
            step = max(1, REFINE_PIXELS // (sizes[-1][0] * sizes[-1][1]))
            for c0 in range(0, len(idx), step):
                chunk = np.array(idx[c0:c0 + step])
                live = np.arange(len(chunk))
                for lv, sk in enumerate(sizes):
                    A = torch.stack([L1[k] for k in chunk[live]])
                    B = torch.stack([L2[k] for k in chunk[live]])
                    Wk = torch.from_numpy(to_level(H[chunk[live]], s1, s2, sk)).to(A.device)
                    W, r, _, st = ops.find_homography_ecc_split(_level_plane(B, sk), _level_plane(A, sk), Wk, iters, eps)
                    W, r, st = W.cpu().numpy(), r.cpu().numpy(), st.cpu().numpy()
                    ok = st == 0
                    ks = chunk[live]
                    rho[ks] = r
                    H[ks[ok]] = from_level(W[ok], s1, s2, sk)
                    reached[ks[ok]] = lv + 1
                    status[ks[~ok]] = st[~ok]
                    live = live[ok]
                    if not len(live):
                        break
        e1.record()
        e1.synchronize()
        self.last_ms["refine"] = e0.elapsed_time(e1)
        return H, rho, status, reached


# ---- files --------------------------------------------------------------------------------------------------------------
def decode_images(paths, device="cuda"):
    """Image files -> list of uint8 [h,w,3] RGB CUDA tensors, bit-identical to cv2.imread(path, IMREAD_COLOR)[..., ::-1]:
    baseline JPEG and 8-bit PNG files on the device (one decode launch per format and size, as the loaders' decode plans),
    every other file, and any the device fails on, through cv2.imread.  Raises IOError naming an unreadable file."""
    import cv2
    blobs = []
    for p in paths:
        with open(p, "rb") as f:
            blobs.append(f.read())
    plans = collections.OrderedDict()
    for k, b in enumerate(blobs):
        for kind, parse in (("jpeg", ops.jpeg_parse), ("png", ops.png_parse)):
            info = parse(b)
            if info.reason == 0:
                plans.setdefault((kind, info.height, info.width), []).append(k)
                break
    out = [None] * len(paths)
    for (kind, h, w), take in plans.items():
        if kind == "jpeg":
            imgs, status = ops.JpegPlan([blobs[k] for k in take], h, w).decode(device)
        else:
            imgs, status = ops.PngPlan([blobs[k] for k in take], h, w).decode(device, rgb=True)
        st = status.cpu().numpy()
        for j, k in enumerate(take):
            if st[j] == 0:
                out[k] = imgs[j]
    for k, p in enumerate(paths):
        if out[k] is None:
            im = cv2.imread(p, cv2.IMREAD_COLOR)
            if im is None:
                raise IOError("cannot read %s" % p)
            out[k] = torch.from_numpy(np.ascontiguousarray(im[..., ::-1])).to(device)
    return out


def read_pairs(path):
    """`img1 img2` per line, paths relative to the list file's directory -> [(img1, img2)] as written, [(path1, path2)]."""
    base = os.path.dirname(os.path.abspath(path))
    names = []
    with open(path) as f:
        for ln in f:
            parts = ln.split()
            if not parts:
                continue
            if len(parts) != 2:
                raise ValueError("%s: expected 'img1 img2', got %r" % (path, ln.rstrip("\n")))
            names.append((parts[0], parts[1]))
    return names, [(os.path.join(base, a), os.path.join(base, b)) for a, b in names]


def homography_as_written(H):
    """The nine entries of H as homographies.txt stores them: float32 values, written '%.9g', which reads back as float32
    to the same values."""
    return np.asarray(H, np.float64).reshape(-1, 9).astype(np.float32)


def format_line(name1, name2, H):
    return " ".join([name1, name2] + ["%.9g" % v for v in homography_as_written(H)[0]])
