"""Input pipeline with the reference Dataloader's contract (code/dataloader.py:11-22,76-235).

Produces, per batch, the nine post-dataloader tensors the model consumes (`*_batch` attributes / dict keys):
I1, I2, I1_aug, I2_aug [B,P,P,1]; I (=I_aug), I_prime (=I_prime_aug) [B,Hh,W,3]; pts1, gt [B,8]; patch_indices [B,P*P].
JPEG decode runs on the device for the baseline files cv2.imwrite produces, and PNG decode for 8-bit non-interlaced gray,
RGB and RGBA files (both bit-identical to cv2.imread; other files are decoded on the host); list parsing runs on the host; photometric augmentation, normalisation, gray conversion and patch
gather run on the device.  The real-data set (extended_dataloader_params) takes the same device path at its two file sizes,
with its augment + normalise + AREA resize in one kernel, bit-identical to its host path (_disk_batch_extended_host).
`synthetic=N` replaces the on-disk set by N
on-device generated pairs (synthetic.make_batch) — MS-COCO is not available offline.
"""
import os
import time
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


def _value_table(g=None, br=None, c=None):
    """[256, 3] fp32: the real-data host path's augment (g, br, c; none when g is None) and normalise expression evaluated
    on the values 0..255.  Every step is elementwise in the uint8 value and the channel, so a lookup equals it bit for bit."""
    v = np.repeat(np.arange(256, dtype=np.float32)[:, None], 3, axis=1)
    if g is not None:
        v = np.clip(v ** np.float32(g) * np.float32(br) * c, 0, 255)
    return (v - np.array(synthetic.MEAN_I, np.float32)) / np.array(synthetic.STD_I, np.float32)


def normalise_resize_host(t, img_h, img_w):
    """The real-data host path's normalise + cv2 INTER_AREA resize of one fp32 [h,w,3] RGB image to the network size."""
    import cv2
    n = (t - np.array(synthetic.MEAN_I, np.float32)) / np.array(synthetic.STD_I, np.float32)
    return cv2.resize(n, (img_w, img_h), interpolation=cv2.INTER_AREA) if t.shape[:2] != (img_h, img_w) else n


def gather_patches(I_pl, Ip_pl, I_aug, Ip_aug, pts1, P, W):
    """The real-data device path's patch step: patch_indices from each sample's first corner of pts1 [B,8] (CUDA fp32) and
    the gray (channel-mean) P x P patches of the four network-size planes [B,Hh,W,3]."""
    B, dev = pts1.shape[0], pts1.device
    x0 = pts1[:, 0].long(); y0 = pts1[:, 1].long()
    yy, xx = torch.meshgrid(torch.arange(P, device=dev), torch.arange(P, device=dev), indexing="ij")
    pidx = ((yy[None] + y0[:, None, None]) * W + (xx[None] + x0[:, None, None])).reshape(B, -1)
    g = lambda a: torch.gather(a.mean(dim=3).reshape(B, -1), 1, pidx).reshape(B, P, P, 1).contiguous()
    return dict(I1=g(I_pl), I2=g(Ip_pl), I1_aug=g(I_aug), I2_aug=g(Ip_aug), I_aug=I_aug, I_prime_aug=Ip_aug,
                pts1=pts1, gt=None, patch_indices=pidx.to(torch.int32).contiguous())


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
        self._reader, self._pending, self._ready = None, None, []
        self.decode_stats = dict(groups=0, read_s=0.0, wait_s=0.0, group_s=0.0, device_images=0, host_images=0, decode_errors=0, png_images=0)
        if not self.synthetic_pairs:
            self.names, self.pts1, self.gt = read_img_and_gt(params.filenames_file, params.pts1_file, params.gt_file)
            self.num_samples = len(self.names)
            self._order = np.arange(self.num_samples)
            self._cursor = self.num_samples
        else:
            self.num_samples = self.synthetic_pairs

    # ---- on-disk path -------------------------------------------------------------------------------------------
    def _pair_paths(self, idx):
        name = self.names[idx][1] if len(self.names[idx]) > 1 else self.names[idx][0]   # dataloader.py:143-144 (column 1 for both)
        return [os.path.join(self.params.data_path, sub, name) for sub in ("I", "I_prime")]

    def _read_image(self, path, size=None):
        """The host decode: cv2.imread + BGR -> RGB, INTER_AREA-resized to `size` (default: the network size) when it differs."""
        import cv2
        h, w = size or (self.params.img_h, self.params.img_w)
        im = cv2.imread(path, cv2.IMREAD_COLOR)
        if im is None:
            raise IOError("cannot read %s" % path)
        im = cv2.cvtColor(im, cv2.COLOR_BGR2RGB)
        if im.shape[0] != h or im.shape[1] != w:
            im = cv2.resize(im, (w, h), interpolation=cv2.INTER_AREA)    # dataloader.py:245
        return im

    def _read_pair(self, idx):
        return [self._read_image(path) for path in self._pair_paths(idx)]

    def _next_indices(self, B):
        out = []
        while len(out) < B:
            if self._cursor >= self.num_samples:
                if self.shuffle:
                    self._rng.shuffle(self._order)
                self._cursor = 0
            out.append(self._order[self._cursor]); self._cursor += 1
        return np.array(out)

    def _disk_batch_extended_host(self):
        """Real-data samples (code/dataloader.py:146-200): FULL-size images are read, augmented and normalised at full
        size, then AREA-resized to the network size; the ground truth (test only) is four hand-picked correspondences
        (16 numbers), not a 4-point displacement.  JPEG decode, augmentation and resize run on the host as in the reference.
        _disk_batch_extended gives the same batches from the device; this path serves the geometries it does not restate."""
        import cv2
        p = self.params
        B, P, Hh, W, FH, FW = p.batch_size, p.patch_size, p.img_h, p.img_w, p.full_img_h, p.full_img_w
        idx = self._next_indices(B)
        I_aug = np.empty((B, Hh, W, 3), np.float32); Ip_aug = np.empty_like(I_aug); I_pl = np.empty_like(I_aug); Ip_pl = np.empty_like(I_aug)
        full_I = np.empty((B, FH, FW, 3), np.uint8); full_Ip = np.empty_like(full_I)
        aug_tab = np.zeros((B, 11), np.float32)
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
                aug_tab[j, :6] = [1.0, g, br, *c]
                if self.mode != 'train':
                    g, br, c = draw()                                                             # disjoint noise in test
                ba = np.clip(b ** np.float32(g) * np.float32(br) * c, 0, 255)
                aug_tab[j, 6:] = [g, br, *c]
            rs = lambda t: normalise_resize_host(t, Hh, W)
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
        out.update(I_u8=t(full_I), I_prime_u8=t(full_Ip), aug=t(aug_tab))
        self._extended_gt(out, idx)
        return out

    def _extended_gt(self, out, idx):
        if self.gt is not None:
            if self.gt.shape[1] == 16:
                out["gt_corr"] = self.gt[idx].astype(np.float32)                                  # four correspondences (test set)
            else:
                out["gt"] = torch.tensor(self.gt[idx], dtype=torch.float32, device=self.device)

    # The same batches from the device: the full-size uint8 images come from the decode groups below (files at the network
    # size are decoded at that size and brought up to the full size by udh_resize_area_up_u8), and udh_real_prep turns them
    # into the four network-size fp32 images through per-sample value tables.  The tables are the host path's augment +
    # normalise expression evaluated on 0..255, drawn from the RNG in the host path's order.  The channel mean and the
    # patch gather are the host path's torch calls on the same device tensors.
    def _extended_on_device(self):
        """Whether udh_real_prep restates this geometry's fp32 resize (else every batch takes the host path)."""
        p = self.params
        from . import ops
        return (p.full_img_h, p.full_img_w) == (p.img_h, p.img_w) or ops.area_is_generic(p.full_img_h, p.full_img_w, p.img_h, p.img_w)

    def _decode_sizes(self):
        """File sizes the device decoder takes: the full size, and the network size when it can be upscaled on the device."""
        p = self.params
        if not hasattr(p, "full_img_h"):
            return [(p.img_h, p.img_w)]
        sizes = [(p.full_img_h, p.full_img_w)]
        if p.img_h < p.full_img_h and p.img_w < p.full_img_w:
            sizes.append((p.img_h, p.img_w))
        return sizes

    def _draw_batch_extended(self):
        """Indices, value tables [B,4,256,3] (plain I, plain I', augmented I, augmented I') and the [B,11] augmentation
        table, drawn as _disk_batch_extended_host draws: per sample uniform(0, 1), then (g, br, c[3]) when augmenting and
        a second (g, br, c[3]) in test mode."""
        p = self.params
        B = p.batch_size
        idx = self._next_indices(B)
        plain = _value_table()
        tables = np.empty((B, 4, 256, 3), np.float32)
        tables[:] = plain[None, None]
        aug = np.zeros((B, 11), np.float32)
        for j in range(B):
            if self._rng.uniform(0, 1) > (1 - p.do_augment):                                      # dataloader.py:163-169
                draw = lambda: (self._rng.uniform(0.8, 1.2), self._rng.uniform(0.5, 2.0), self._rng.uniform(0.8, 1.2, size=3).astype(np.float32))
                g, br, c = draw()
                tables[j, 2] = _value_table(g, br, c)
                aug[j, :6] = [1.0, g, br, *c]
                if self.mode != 'train':
                    g, br, c = draw()
                tables[j, 3] = _value_table(g, br, c)
                aug[j, 6:] = [g, br, *c]
        return idx, tables, aug

    def _disk_batch_extended(self):
        if not self._extended_on_device():
            return self._disk_batch_extended_host()
        from . import ops
        p = self.params
        B, P, Hh, W = p.batch_size, p.patch_size, p.img_h, p.img_w
        if not self._ready:
            self._decode_group()
        idx, tables, aug, I_u8, Ip_u8 = self._ready.pop(0)
        dev = self.device
        I_pl, Ip_pl, I_aug, Ip_aug = ops.real_prep(I_u8, Ip_u8, torch.from_numpy(tables).to(dev), Hh, W)
        pts1 = torch.tensor(self.pts1[idx], dtype=torch.float32, device=dev)
        out = gather_patches(I_pl, Ip_pl, I_aug, Ip_aug, pts1, P, W)
        out.update(full_I=I_u8.cpu().numpy(), full_I_prime=Ip_u8.cpu().numpy())
        out.update(I_u8=I_u8, I_prime_u8=Ip_u8, aug=torch.from_numpy(aug).to(dev))
        self._extended_gt(out, idx)
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

    # Device decode of the on-disk set.  A group of DECODE_BATCHES batches is decoded in one launch: the indices and the
    # augmentation table of each batch are drawn from the host RNG batch after batch, exactly as the host path draws them,
    # so the batches are the same whichever decoder ran.  A background thread reads (and parses) the next group's files
    # while the current group is being consumed.  Baseline JPEG and 8-bit PNG files of a decode size go to a JpegPlan or a
    # PngPlan per size; the files neither device decoder takes (progressive, palette PNG, another size, a decode error, ...)
    # go through _read_image.  Because a group is built at once, a missing or unreadable file raises
    # its IOError when the first batch of its group is requested (up to DECODE_BATCHES - 1 batches before its own).
    # decode_stats counts, over the loader's life, the groups, the reader thread's seconds, the seconds next_batch spent
    # waiting for it, the seconds next_batch spent building groups (wait included), and the images decoded on the device, on the host, and sent to the host after a device decode error;
    # png_images counts the device-decoded images that were PNG files.
    # DECODE_BATCHES: see DESIGN §4.
    DECODE_BATCHES = 4

    def _draw_batch(self):
        p = self.params
        B = p.batch_size
        idx = self._next_indices(B)
        # augmentation parameters on the host RNG (reproducible order), applied by the fused device kernel
        aug = np.zeros((B, 11), np.float32)
        aug[:, 0] = self._rng.uniform(0, 1, size=B) > (1 - p.do_augment)                          # dataloader.py:163-169
        draw = lambda: np.concatenate([[self._rng.uniform(0.8, 1.2), self._rng.uniform(0.5, 2.0)], self._rng.uniform(0.8, 1.2, size=3)])
        for j in range(B):
            a = draw()
            aug[j, 1:6] = a
            aug[j, 6:11] = a if self.mode == 'train' else draw()                                   # joint (train) / disjoint (test)
        return idx, aug

    def _read_group(self, paths, sizes):
        """Background thread: file bytes -> ([(size, device-decodable file positions, JpegPlan or PngPlan)] per format and
        size in `sizes` that has files).  File reads and the ctypes parser calls release the GIL."""
        from . import ops
        t0 = time.perf_counter()
        kinds = ((ops.jpeg_parse, ops.JpegPlan), (ops.png_parse, ops.PngPlan))
        blobs = [{s: [] for s in sizes} for _ in kinds]
        take = [{s: [] for s in sizes} for _ in kinds]
        for k, path in enumerate(paths):
            try:
                with open(path, "rb") as f:
                    b = f.read()
            except OSError:
                continue                                       # _read_image raises the host path's error
            for j, (parse, _) in enumerate(kinds):
                info = parse(b)
                if info.reason == 0:
                    if (info.height, info.width) in blobs[j]:
                        blobs[j][(info.height, info.width)].append(b); take[j][(info.height, info.width)].append(k)
                    break
        plans = [(s, take[j][s], plan(blobs[j][s], *s)) for j, (_, plan) in enumerate(kinds) for s in sizes if blobs[j][s]]
        return plans, time.perf_counter() - t0

    def _submit_group(self):
        extended = hasattr(self.params, "full_img_h")
        draws = [self._draw_batch_extended() if extended else self._draw_batch() for _ in range(self.DECODE_BATCHES)]
        paths = [path for d in draws for i in d[0] for path in self._pair_paths(i)]
        if self._reader is None:
            import concurrent.futures
            self._reader = concurrent.futures.ThreadPoolExecutor(max_workers=1, thread_name_prefix="udh-jpeg-reader")
        return draws, paths, self._reader.submit(self._read_group, paths, self._decode_sizes())

    def _decode_group(self):
        t_group = time.perf_counter()
        if self._pending is None:
            self._pending = self._submit_group()
        draws, paths, fut = self._pending
        self._pending = self._submit_group()                   # read the next group while this one is decoded and consumed
        t0 = time.perf_counter()
        plans, read_s = fut.result()
        st = self.decode_stats
        st["groups"] += 1; st["read_s"] += read_s; st["wait_s"] += time.perf_counter() - t0
        p, dev = self.params, self.device
        h, w = self._decode_sizes()[0]                          # the size the batch is assembled at
        imgs = torch.empty(len(paths), h, w, 3, dtype=torch.uint8, device=dev)
        host = set(range(len(paths)))
        from . import ops
        for size, take, plan in plans:
            png = isinstance(plan, ops.PngPlan)
            out, status = plan.decode(dev, rgb=True) if png else plan.decode(dev)      # RGB, as _read_image returns
            if size != (h, w):
                out = ops.resize_area_up_u8(out, h, w)           # network-size files of the real-data set
            imgs[torch.tensor(take, device=dev)] = out
            bad = [take[k] for k in np.flatnonzero(status.cpu().numpy())]
            host = (host - set(take)) | set(bad)
            st["device_images"] += len(take) - len(bad); st["decode_errors"] += len(bad)
            if png:
                st["png_images"] += len(take) - len(bad)
        host = sorted(host)
        st["host_images"] += len(host)
        if host:
            hi = np.stack([self._read_image(paths[k], (h, w)) for k in host])
            imgs[torch.tensor(host, device=dev)] = torch.from_numpy(hi).to(dev)
        imgs = imgs.view(len(draws), p.batch_size, 2, h, w, 3)
        self._ready = [tuple(d) + (imgs[k, :, 0].contiguous(), imgs[k, :, 1].contiguous()) for k, d in enumerate(draws)]
        st["group_s"] += time.perf_counter() - t_group

    def _disk_batch(self):
        p = self.params
        B, P, Hh, W = p.batch_size, p.patch_size, p.img_h, p.img_w
        if 'normalize' not in p.augment_list:
            raise NotImplementedError("augment_list without 'normalize' is not supported (the reference default is ['normalize'])")
        if not self._ready:
            self._decode_group()
        idx, aug, I_u8, Ip_u8 = self._ready.pop(0)
        dev = self.device
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
