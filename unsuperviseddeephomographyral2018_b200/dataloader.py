"""Input pipeline with the reference Dataloader's contract (code/dataloader.py:11-22,76-235).

Produces, per batch, the nine post-dataloader tensors the model consumes (`*_batch` attributes / dict keys):
I1, I2, I1_aug, I2_aug [B,P,P,1]; I (=I_aug), I_prime (=I_prime_aug) [B,Hh,W,3]; pts1, gt [B,8]; patch_indices [B,P*P].
JPEG decode and list parsing run on the host (as in the reference: queue-runner threads); photometric augmentation,
normalisation, gray conversion and patch gather run on the device.  `synthetic=N` replaces the on-disk set by N
on-device generated pairs (synthetic.make_batch) — MS-COCO is not available offline.
"""
import os
from collections import namedtuple

import numpy as np
import torch

from . import synthetic

dataloader_params = namedtuple('parameters',
                               'data_path,'
                               'filenames_file,'
                               'pts1_file,'
                               'gt_file,'
                               'mode,'
                               'batch_size,'
                               'img_h,'
                               'img_w,'
                               'patch_size,'
                               'augment_list,'
                               'do_augment,')


# real-data set: a sample consists of full-size images, network-size images and the patch (code/dataloader.py:26-39)
extended_dataloader_params = namedtuple('extended_parameters',
                                        'data_path,'
                                        'filenames_file,'
                                        'pts1_file,'
                                        'gt_file,'
                                        'mode,'
                                        'batch_size,'
                                        'img_h,'
                                        'img_w,'
                                        'patch_size,'
                                        'augment_list,'
                                        'do_augment,'
                                        'full_img_h,'
                                        'full_img_w')


def count_text_lines(path):
    """utils/utils.py:358-362."""
    with open(path, 'r') as f:
        return len(f.readlines())


def read_img_and_gt(filenames_file, pts1_file, gt_file):
    """dataloader.py:49-72: list lines "<I name> <I' name>", pts1 / gt = 8 floats per line (np.savetxt)."""
    with open(pts1_file, 'r') as f:
        pts1 = np.array([ln.split() for ln in f.read().strip().split("\n")]).astype('float64')
    with open(filenames_file, 'r') as f:
        names = [ln.split() for ln in f.read().strip().split("\n")]
    if not gt_file:
        return names, pts1, None
    with open(gt_file, 'r') as f:
        gt = np.array([ln.split() for ln in f.read().strip().split("\n")]).astype('float64')
    return names, pts1, gt


class Dataloader(object):
    def __init__(self, params, shuffle=True, synthetic_pairs=0, seed=0, device="cuda", rho=45):
        self.params = params
        self.mode = params.mode
        self.shuffle = shuffle
        self.device = torch.device(device)
        self.synthetic_pairs = int(synthetic_pairs)
        self.seed = seed
        self.rho = rho
        self._rng = np.random.default_rng(seed)
        self._step = 0
        if not self.synthetic_pairs:
            self.names, self.pts1, self.gt = read_img_and_gt(params.filenames_file, params.pts1_file, params.gt_file)
            self.num_samples = len(self.names)
            self._order = np.arange(self.num_samples)
            self._cursor = self.num_samples
        else:
            self.num_samples = self.synthetic_pairs

    # ---- on-disk path -------------------------------------------------------------------------------------------
    def _read_pair(self, idx):
        import cv2
        name = self.names[idx][1] if len(self.names[idx]) > 1 else self.names[idx][0]   # dataloader.py:143-144 (column 1 for both)
        imgs = []
        for sub in ("I", "I_prime"):
            im = cv2.imread(os.path.join(self.params.data_path, sub, name), cv2.IMREAD_COLOR)
            if im is None:
                raise IOError("cannot read %s" % os.path.join(self.params.data_path, sub, name))
            im = cv2.cvtColor(im, cv2.COLOR_BGR2RGB)
            if im.shape[0] != self.params.img_h or im.shape[1] != self.params.img_w:
                im = cv2.resize(im, (self.params.img_w, self.params.img_h), interpolation=cv2.INTER_AREA)    # dataloader.py:245
            imgs.append(im)
        return imgs

    def _next_indices(self, B):
        out = []
        while len(out) < B:
            if self._cursor >= self.num_samples:
                if self.shuffle:
                    self._rng.shuffle(self._order)
                self._cursor = 0
            out.append(self._order[self._cursor]); self._cursor += 1
        return np.array(out)

    def _disk_batch_extended(self):
        """Real-data samples (code/dataloader.py:146-200): FULL-size images are read, augmented and normalised at full
        size, then AREA-resized to the network size; the ground truth (test only) is four hand-picked correspondences
        (16 numbers), not a 4-point displacement.  JPEG decode, augmentation and resize run on the host as in the reference."""
        import cv2
        p = self.params
        B, P, Hh, W, FH, FW = p.batch_size, p.patch_size, p.img_h, p.img_w, p.full_img_h, p.full_img_w
        idx = self._next_indices(B)
        mean, std = np.array(synthetic.MEAN_I, np.float32), np.array(synthetic.STD_I, np.float32)
        I_aug = np.empty((B, Hh, W, 3), np.float32); Ip_aug = np.empty_like(I_aug); I_pl = np.empty_like(I_aug); Ip_pl = np.empty_like(I_aug)
        full_I = np.empty((B, FH, FW, 3), np.uint8); full_Ip = np.empty_like(full_I)
        for j, i in enumerate(idx):
            name = self.names[i][1] if len(self.names[i]) > 1 else self.names[i][0]
            pair = []
            for sub in ("I", "I_prime"):
                im = cv2.imread(os.path.join(p.data_path, sub, name), cv2.IMREAD_COLOR)
                if im is None:
                    raise IOError("cannot read %s" % os.path.join(p.data_path, sub, name))
                im = cv2.cvtColor(im, cv2.COLOR_BGR2RGB)
                if im.shape[0] != FH or im.shape[1] != FW:
                    im = cv2.resize(im, (FW, FH), interpolation=cv2.INTER_AREA)
                pair.append(im)
            full_I[j], full_Ip[j] = pair
            a, b = pair[0].astype(np.float32), pair[1].astype(np.float32)
            aa, ba = a, b
            if self._rng.uniform(0, 1) > (1 - p.do_augment):                                      # :163-169
                draw = lambda: (self._rng.uniform(0.8, 1.2), self._rng.uniform(0.5, 2.0), self._rng.uniform(0.8, 1.2, size=3).astype(np.float32))
                g, br, c = draw()
                aa = np.clip(a ** np.float32(g) * np.float32(br) * c, 0, 255)
                if self.mode != 'train':
                    g, br, c = draw()                                                             # disjoint noise in test
                ba = np.clip(b ** np.float32(g) * np.float32(br) * c, 0, 255)
            rs = lambda t: cv2.resize((t - mean) / std, (W, Hh), interpolation=cv2.INTER_AREA) if (FH != Hh or FW != W) else (t - mean) / std
            I_pl[j], Ip_pl[j], I_aug[j], Ip_aug[j] = rs(a), rs(b), rs(aa), rs(ba)
        dev = self.device
        pts1 = torch.tensor(self.pts1[idx], dtype=torch.float32, device=dev)
        x0 = pts1[:, 0].long(); y0 = pts1[:, 1].long()
        yy, xx = torch.meshgrid(torch.arange(P, device=dev), torch.arange(P, device=dev), indexing="ij")
        pidx = ((yy[None] + y0[:, None, None]) * W + (xx[None] + x0[:, None, None])).reshape(B, -1)
        t = lambda a: torch.from_numpy(a).to(dev)
        g = lambda a: torch.gather(t(a).mean(dim=3).reshape(B, -1), 1, pidx).reshape(B, P, P, 1).contiguous()
        out = dict(I1=g(I_pl), I2=g(Ip_pl), I1_aug=g(I_aug), I2_aug=g(Ip_aug), I_aug=t(I_aug).contiguous(), I_prime_aug=t(Ip_aug).contiguous(),
                   pts1=pts1, gt=None, patch_indices=pidx.to(torch.int32).contiguous(), full_I=full_I, full_I_prime=full_Ip)
        if self.gt is not None:
            if self.gt.shape[1] == 16:
                out["gt_corr"] = self.gt[idx].astype(np.float32)                                  # four correspondences (test set)
            else:
                out["gt"] = torch.tensor(self.gt[idx], dtype=torch.float32, device=dev)
        return out

    def _synthetic_real_batch(self):
        """Stand-in for the (private) aerial data at the real-data geometry (142x190 images, 128 patches): on-device
        synthetic pairs; training batches carry NO ground truth (gt-less l1 training), test batches carry four
        correspondences per pair in the frame the reference clicked them on (2x the full image)."""
        p = self.params
        rho = min(self.rho, (p.img_h - p.patch_size) // 2, (p.img_w - p.patch_size) // 2)
        b = synthetic.make_batch_fast(p.batch_size, seed=self.seed * 1000003 + self._step, img_h=p.img_h, img_w=p.img_w, patch=p.patch_size,
                                      rho=rho, device=self.device, do_augment=float(p.do_augment), mode=self.mode)
        if self.mode != 'train':
            from . import real_metrics as rm
            r = float(p.full_img_h) / float(p.img_h)
            rng = np.random.default_rng(self.seed * 7 + self._step)
            pts1, gt = b["pts1"].cpu().numpy().astype(np.float64), b["gt"].cpu().numpy().astype(np.float64)
            corr = np.zeros((p.batch_size, 16), np.float32)
            for j in range(p.batch_size):
                H = rm.get_perspective_transform((pts1[j].reshape(4, 2) * r).astype(np.float32), ((pts1[j] + gt[j]).reshape(4, 2) * r).astype(np.float32))
                c1 = np.stack([rng.uniform(40, p.full_img_w - 40, 4), rng.uniform(40, p.full_img_h - 40, 4)], 1)
                c2 = rm.perspective_transform(c1, np.linalg.inv(H))
                corr[j] = np.concatenate([c1.reshape(-1), c2.reshape(-1)]) * 2.0                 # clicked on 480x640 frames
            b["gt_corr"] = corr
        b["gt_4pt"] = b["gt"]
        b["gt"] = None                                                                            # the real path never sees a 4-point gt
        return b

    def _disk_batch(self):
        p = self.params
        B, P, Hh, W = p.batch_size, p.patch_size, p.img_h, p.img_w
        idx = self._next_indices(B)
        I = np.empty((B, Hh, W, 3), np.uint8); Ip = np.empty_like(I)
        for j, i in enumerate(idx):
            I[j], Ip[j] = self._read_pair(i)
        dev = self.device
        I_u8 = torch.from_numpy(I).to(dev); Ip_u8 = torch.from_numpy(Ip).to(dev)
        if 'normalize' not in p.augment_list:
            raise NotImplementedError("augment_list without 'normalize' is not supported (the reference default is ['normalize'])")
        # augmentation parameters on the host RNG (reproducible order), applied by the fused device kernel
        aug = np.zeros((B, 11), np.float32)
        aug[:, 0] = self._rng.uniform(0, 1, size=B) > (1 - p.do_augment)                          # dataloader.py:163-169
        draw = lambda: np.concatenate([[self._rng.uniform(0.8, 1.2), self._rng.uniform(0.5, 2.0)], self._rng.uniform(0.8, 1.2, size=3)])
        for j in range(B):
            a = draw()
            aug[j, 1:6] = a
            aug[j, 6:11] = a if self.mode == 'train' else draw()                                   # joint (train) / disjoint (test)
        pts1 = torch.tensor(self.pts1[idx], dtype=torch.float32, device=dev)
        gt = torch.tensor(self.gt[idx], dtype=torch.float32, device=dev) if self.gt is not None else None
        aug_dev = torch.tensor(aug, device=dev)
        out = synthetic.prep_u8(I_u8, Ip_u8, pts1, aug_dev, P, want_rgb=True)
        out["gt"] = gt
        out.update(I_u8=I_u8, I_prime_u8=Ip_u8, aug=aug_dev)       # the decoded images and their augmentation (direct-method baseline)
        out["I_aug"] = out.pop("I_aug_rgb")                        # the reference contract: [B,Hh,W,3] normalised (augmented) I
        return out

    # ---- public ---------------------------------------------------------------------------------------------------
    def next_batch(self):
        p = self.params
        extended = hasattr(p, "full_img_h")
        if extended:
            b = self._synthetic_real_batch() if self.synthetic_pairs else self._disk_batch_extended()
        elif self.synthetic_pairs:
            # on-device generator + fused augment / normalise / gray / crop (four kernel launches per batch); photometric
            # augmentation as the reference: probability do_augment, joint in train, disjoint in test
            b = synthetic.make_batch_fast(p.batch_size, seed=self.seed * 1000003 + self._step, img_h=p.img_h, img_w=p.img_w,
                                          patch=p.patch_size, rho=self.rho, device=self.device, do_augment=float(p.do_augment),
                                          mode=self.mode)
        else:
            b = self._disk_batch()
        self._step += 1
        # the reference's attribute names
        self.I1_batch, self.I2_batch, self.I1_aug_batch, self.I2_aug_batch = b["I1"], b["I2"], b["I1_aug"], b["I2_aug"]
        self.I_batch, self.I_prime_batch = b["I_aug"], b["I_prime_aug"]
        self.pts1_batch, self.gt_batch, self.patch_indices_batch = b["pts1"], b["gt"], b["patch_indices"]
        return b
