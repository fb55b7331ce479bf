"""Restatement of the fp32 CUDA-core engine's arithmetic (UDH_NUMERIC_FP32, csrc/cnn_simt.cu) — TEST INFRASTRUCTURE ONLY.

The engine's kernels are fixed sequences of fp32 operations, so chosen outputs can be recomputed bit for bit:
  * `conv3x3_kernel`: one thread owns an output element and accumulates with `fmaf`, starting from +0, over input channel
    (in chunks of CK consecutive channels, which keeps plain channel order), ky, kx, zero padding included; then one fp32
    `+ bias` (+0 without a bias), `fmaxf(v, 0)` for ReLU, and `mask_src > 0 ? v : 0`.  The dgrad is the same kernel on the
    rotated weights wrot[ky][kx][co][ci] = w[2-ky][2-kx][ci][co].  `conv_chain` repeats that for chosen elements.
  * `wgrad3x3_kernel`: CTA x of the reported partition walks the 8x16 pixel tiles [x per, (x+1) per) in (n, tile row,
    tile column) order; its thread for row phase s sums rows s, s + split, ... of each tile, columns 0..15, with one `fmaf`
    per pixel (db: one fp32 add per pixel), and adds the partial to dW with `atomicAdd`.  `wgrad_partials` /
    `bias_partials` give every partial of chosen elements; the atomics add them in an unknown order, which is bounded, not
    restated (`sum_bound`).
  * `maxpool_fwd_kernel` / `maxpool_bwd_kernel`: the maximum of each 2x2 window; the gradient goes to the FIRST maximum in
    row-major window order, and only when that maximum is > 0 (`pool_fwd`, `pool_bwd`).
fmaf is `oracle.warp_fp32.fmaf32`.  Arrays are NumPy; the gathers also accept torch tensors (on any device), so a test can
pick operands out of device activations without copying them whole.
"""
import numpy as np
import torch

from .warp_fp32 import U32, f32, fmaf32

TH, TW = 8, 16        # pixel tile of the conv / wgrad kernels (rows x columns)


def gamma(n, u=U32):
    """gamma_n = n u / (1 - n u): the relative bound of n rounded operations in a sum (Higham, Lemma 3.1)."""
    n = np.asarray(n, dtype=np.float64)
    return n * u / (1.0 - n * u)


def _np(a):
    return a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


def _take(x, n, yy, xx, c):
    """x[n, yy, xx, c] with +0 outside the image (the kernels' zero halo); index arrays broadcast, result float32 NumPy."""
    H, W = x.shape[1], x.shape[2]
    n, yy, xx, c = np.broadcast_arrays(*(np.asarray(v, dtype=np.int64) for v in (n, yy, xx, c)))
    ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
    yc, xc = np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)
    if isinstance(x, torch.Tensor):
        t = lambda a: torch.as_tensor(a, device=x.device)
        v = x[t(n), t(yc), t(xc), t(c)].detach().cpu().numpy()
    else:
        v = x[n, yc, xc, c]
    return np.where(ok, v, f32(0)).astype(f32)


def _stack_planes(x, x2):
    if x2 is None:
        return x
    if isinstance(x, torch.Tensor):
        return torch.stack([x.reshape(x.shape[:3]), x2.reshape(x2.shape[:3])], dim=3)
    return np.stack([np.asarray(x).reshape(x.shape[:3]), np.asarray(x2).reshape(x2.shape[:3])], axis=3)


def conv_operands(x, w, n, y, xx, o, dgrad=False, x2=None):
    """The (input, weight) pairs of output elements (n, y, xx, o) in the kernel's accumulation order: [S, 9 kin] each.
    Forward: x [B,H,W,cin] (or the planes x, x2), w [3,3,cin,cout], o = output channel.  dgrad: x = g [B,H,W,cout], w the
    layer's [3,3,cin,cout] kernel, o = the layer's input channel."""
    x = _stack_planes(x, x2)
    w = _np(w).astype(f32)
    wk = w[::-1, ::-1].transpose(0, 1, 3, 2) if dgrad else w          # [3,3,kin,kout] of the conv the kernel runs
    kin = wk.shape[2]
    c, ky, kx = (a.reshape(-1) for a in np.meshgrid(np.arange(kin), np.arange(3), np.arange(3), indexing="ij"))
    n, y, xx, o = (np.asarray(v, dtype=np.int64)[:, None] for v in (n, y, xx, o))
    a = _take(x, n, y + ky[None] - 1, xx + kx[None] - 1, c[None])
    b = wk[ky[None], kx[None], c[None], o]
    return a, np.ascontiguousarray(b, dtype=f32)


def conv_chain(x, w, n, y, xx, o, bias=None, relu=False, mask=None, dgrad=False, x2=None):
    """conv3x3_kernel's value of output elements (n, y, xx, o), bit for bit: the fmaf chain, + bias, ReLU, mask."""
    a, b = conv_operands(x, w, n, y, xx, o, dgrad, x2)
    acc = np.zeros(a.shape[0], f32)
    for k in range(a.shape[1]):
        acc = fmaf32(a[:, k], b[:, k], acc)
    bv = _np(bias).astype(f32)[np.asarray(o)] if bias is not None else f32(0)
    v = (acc + bv).astype(f32)
    if relu:
        v = np.maximum(v, f32(0))
    if mask is not None:
        v = np.where(_take(mask, n, y, xx, o) > 0, v, f32(0)).astype(f32)
    return v


def _partial_terms(B, H, W, part):
    """Pixel (n, y, x) of step j of every partial (cta, s): [m, L] int arrays and a validity mask (the last CTA's range can
    end early).  part = (ctas_x, tiles_per_cta, row_split)."""
    ctas, per, split = part
    rows = TH // split
    tiles_x, tiles_img = W // TW, (W // TW) * (H // TH)
    j = np.arange(per * rows * TW)
    cta, s = np.repeat(np.arange(ctas), split), np.tile(np.arange(split), ctas)
    t = cta[:, None] * per + j[None] // (rows * TW)
    r = s[:, None] + split * ((j[None] // TW) % rows)
    c = np.broadcast_to(j[None] % TW, t.shape)
    ok = t < B * tiles_img
    t = np.where(ok, t, 0)
    nn, tt = t // tiles_img, t % tiles_img
    return nn, (tt // tiles_x) * TH + r, (tt % tiles_x) * TW + c, ok


def wgrad_partials(x, g, part, ky, kx, ci, co, x2=None):
    """Every thread partial of dW[ky, kx, ci, co] (chosen elements, arrays of E): float32 [E, ctas_x row_split], in (CTA,
    row phase) order; x [B,H,W,cin] (or the planes x, x2), g [B,H,W,cout]."""
    x = _stack_planes(x, x2)
    B, H, W = g.shape[0], g.shape[1], g.shape[2]
    nn, yy, xx, ok = _partial_terms(B, H, W, part)
    e = lambda v: np.asarray(v, dtype=np.int64)[:, None, None]
    a = _take(x, nn[None], yy[None] + e(ky) - 1, xx[None] + e(kx) - 1, e(ci))
    b = _take(g, nn[None], yy[None], xx[None], e(co))
    acc = np.zeros(a.shape[:2], f32)
    for j in range(a.shape[2]):
        acc = np.where(ok[None, :, j], fmaf32(a[:, :, j], b[:, :, j], acc), acc).astype(f32)
    return acc


def bias_partials(g, part, co):
    """Every thread partial of db[co] (chosen channels): float32 [E, ctas_x row_split], plain fp32 adds."""
    B, H, W = g.shape[0], g.shape[1], g.shape[2]
    nn, yy, xx, ok = _partial_terms(B, H, W, part)
    b = _take(g, nn[None], yy[None], xx[None], np.asarray(co, dtype=np.int64)[:, None, None])
    acc = np.zeros(b.shape[:2], f32)
    for j in range(b.shape[2]):
        acc = np.where(ok[None, :, j], acc + b[:, :, j], acc).astype(f32)
    return acc


def sum_bound(partials):
    """(float64 sum, bound) of fp32 partials added into a +0 accumulator in ANY order: |fl(sum) - sum| <= gamma_{m-1} sum|p|."""
    p = np.asarray(partials, dtype=np.float64)
    m = p.shape[-1]
    return p.sum(axis=-1), gamma(max(m - 1, 0)) * np.abs(p).sum(axis=-1)


def _windows(x):
    return x[:, 0::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 0::2], x[:, 1::2, 1::2]


def pool_fwd(x):
    """2x2 max of NHWC torch x."""
    a, b, c, d = _windows(x)
    return torch.maximum(torch.maximum(a, b), torch.maximum(c, d))


def pool_bwd(x, dout):
    """The backward rule: dout goes to the first maximum of each window in row-major order, and only when it is > 0; every
    other element gets +0."""
    a, b, c, d = _windows(x)
    m, k = a.clone(), torch.zeros(a.shape, dtype=torch.int8, device=x.device)
    for i, v in ((1, b), (2, c), (3, d)):
        win = v > m
        m = torch.where(win, v, m)
        k = torch.where(win, torch.full_like(k, i), k)
    val = torch.where(m > 0, dout, torch.zeros_like(dout))
    din = torch.zeros_like(x)
    for i, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        din[:, dy::2, dx::2] = torch.where(k == i, val, torch.zeros_like(val))
    return din
