"""NumPy restatement of the device input pipeline of the train step — TEST INFRASTRUCTURE ONLY.

Bit for bit and in kernel order:
  csrc/gen.cu   texture_u8_kernel (the splitmix keys, lattice, smoothstep and octave chain), corners_kernel and
                prep_u8_ex_kernel (the per-sample tables, the gray sum, the patch gather and the origin);
  csrc/prep.cu  normalise_u8_kernel (with its float4 channel phase) and patches_u8_kernel.

The build has no fast-math, so every fp32 operation is IEEE: `/` and `__fdiv_rn` are correctly rounded divisions, and the
only contractions are the ones ptxas chose, read from the SASS of texture_u8_kernel (sm_90a, CUDA 12.9):
  hash_unit        fma(float(h >> 8), 2^-24, -0.5)                         exact either way
  fx, tx, smooth   x * 2^-o, trunc, fx - gx, (tx * tx) * (3 - (tx + tx))   exact: tx has at most 5 fraction bits
  row blends       top = fma(tx, b - a, a), bottom = fma(tx, d - c, c)
  column blend     fma(ty, bottom - top, top)
  octave sum       v = fma(blend, amp_o, v), o = 1 .. 5 in order, amp_o folded to fp32 constants (AMP)
  output           trunc(min(max(fma(v, 9.8, 127.5), 0), 255))
`fmaf32` (oracle/warp_fp32.py) rounds each fma once.

The augmentation's pow is fp64 `pow` rounded once to fp32, the project's definition (common.cuh `denorm_u8`,
oracle/ecc.py, oracle/draw.py).  CUDA's fp64 pow and the host's are each within 2 fp64 ulps of the exact power, so both
round to the same fp32 value unless the power lies that close to an fp32 rounding boundary; `pow_f32` asserts a margin of
64 fp64 ulps, so a table that passes it is the correctly rounded power on either side.
"""
import numpy as np

from .warp_fp32 import fmaf32

f32 = np.float32
u64 = np.uint64
MEAN = np.array([118.93, 113.97, 102.60], f32)
STD = np.array([69.85, 68.81, 72.45], f32)
TAG_CORNERS = 18                 # stream tags: c * 6 + o for the texture lattices, then x0, y0 and the 8 gt draws


def _amps():
    a, out = f32(1.0), []
    for _ in range(5):
        a = f32(a * f32(1.8660660))
        out.append(a)
    return out


AMP = _amps()                    # amp of octaves 1..5: the fp32 product chain the compiler folds


# ---------------------------------------------------------------------------- keys
def mix64(x):
    """splitmix64 (gen.cu `mix64`): the golden-ratio step and the finaliser, modulo 2^64, on uint64 arrays."""
    x = np.array(x, dtype=u64, ndmin=1)
    with np.errstate(over="ignore"):
        x = x + u64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> u64(30))) * u64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> u64(27))) * u64(0x94D049BB133111EB)
    return x ^ (x >> u64(31))


def hash_u32(x):
    return (mix64(x) >> u64(32)).astype(np.uint32)


def hash_unit(x):
    """[-0.5, 0.5): float(h >> 8) * 2^-24 - 0.5, exact."""
    return ((hash_u32(x) >> np.uint32(8)).astype(f32) * f32(2.0 ** -24) - f32(0.5)).astype(f32)


def stream_key(seed, b, tag):
    """gen.cu `stream_key`: mix64(mix64(mix64(seed) ^ b) ^ tag); b and tag broadcast."""
    s = mix64(np.uint64(int(seed) & 0xFFFFFFFFFFFFFFFF))
    b = np.asarray(b, np.int64).astype(np.uint32).astype(u64)
    t = np.asarray(tag, np.int64).astype(np.uint32).astype(u64)
    return mix64(mix64(s ^ b) ^ t)


def lattice(key, gx, gy):
    """Lattice value at integer (gx, gy) of the lattice with stream key `key`."""
    gx = np.asarray(gx, np.int64).astype(np.uint32).astype(u64)
    gy = np.asarray(gy, np.int64).astype(np.uint32).astype(u64)
    return hash_unit(u64(key) ^ (gx | (gy << u64(32))))


# ---------------------------------------------------------------------------- texture_u8_kernel, corners_kernel
def texture(seed, b, Hh, W):
    """Sample b of udh_synth_scene_u8's texture: uint8 [Hh, W, 3]."""
    out = np.empty((Hh, W, 3), np.uint8)
    for c in range(3):
        v = texture_v(seed, b, c, Hh, W)
        out[..., c] = np.trunc(np.clip(fmaf32(v, f32(9.8), f32(127.5)), f32(0), f32(255))).astype(np.uint8)
    return out


def texture_v(seed, b, c, Hh, W):
    """The fp32 octave sum v of channel c of sample b, [Hh, W], before the output scaling."""
    xs = np.arange(W, dtype=np.int64)
    ys = np.arange(Hh, dtype=np.int64)
    keys = stream_key(seed, b, c * 6 + np.arange(6))
    v = lattice(keys[0], xs[None, :], ys[:, None])
    for o in range(1, 6):
        s = f32(1.0 / (1 << o))
        fx = (xs.astype(f32) * s).astype(f32); fy = (ys.astype(f32) * s).astype(f32)
        gx = fx.astype(np.int64); gy = fy.astype(np.int64)                     # (int) truncates; fx >= 0
        tx = (fx - gx.astype(f32)).astype(f32); ty = (fy - gy.astype(f32)).astype(f32)
        tx = ((tx * tx) * (f32(3) - (tx + tx))).astype(f32)
        ty = ((ty * ty) * (f32(3) - (ty + ty))).astype(f32)
        G = lattice(keys[o], np.arange(gx[-1] + 2)[None, :], np.arange(gy[-1] + 2)[:, None])
        a = G[gy[:, None], gx[None, :]]; bb = G[gy[:, None], gx[None, :] + 1]
        cc = G[gy[:, None] + 1, gx[None, :]]; d = G[gy[:, None] + 1, gx[None, :] + 1]
        TX = np.broadcast_to(tx[None, :], a.shape); TY = np.broadcast_to(ty[:, None], a.shape)
        top = fmaf32(TX, (bb - a).astype(f32), a)
        bot = fmaf32(TX, (d - cc).astype(f32), cc)
        v = fmaf32(fmaf32(TY, (bot - top).astype(f32), top), AMP[o - 1], v)
    return v


def corners(seed, B, Hh, W, P, rho):
    """corners_kernel: pts1 [B,8] and gt [B,8] fp32; draw i of sample b is hash_u32(stream_key(seed, b, 18 + i))."""
    b = np.arange(B)
    draw = lambda i: hash_u32(stream_key(seed, b, TAG_CORNERS + i)).astype(np.int64)
    x0 = rho + draw(0) % (W - 2 * rho - P + 1)
    y0 = rho + draw(1) % (Hh - 2 * rho - P + 1)
    pts1 = np.stack([x0, y0, x0 + P, y0, x0 + P, y0 + P, x0, y0 + P], 1).astype(f32)
    gt = np.stack([draw(2 + i) % (2 * rho + 1) - rho for i in range(8)], 1).astype(f32)
    return pts1, gt


def scene(seed, B, Hh, W, P, rho, samples=None):
    """udh_synth_scene_u8: ({b: texture of sample b} for `samples` (default all), pts1, gt)."""
    samples = range(B) if samples is None else samples
    pts1, gt = corners(seed, B, Hh, W, P, rho)
    return {b: texture(seed, b, Hh, W) for b in samples}, pts1, gt


# ---------------------------------------------------------------------------- prep_u8_ex_kernel
def pow_f32(x, g, margin_ulps=64):
    """float32(pow(float64 x, float64 g)) for uint8 values x, asserting that the fp64 power lies at least margin_ulps fp64
    ulps from every fp32 rounding boundary (so any pow within 2 ulps of exact rounds to the same fp32 value)."""
    x64 = np.asarray(x, np.float64)
    p = np.power(x64, np.float64(f32(g)))
    r = p.astype(f32)
    r64 = r.astype(np.float64)
    up = np.nextafter(r, f32(np.inf)).astype(np.float64); dn = np.nextafter(r, f32(-np.inf)).astype(np.float64)
    mid = np.where(p >= r64, (r64 + up) / 2, (r64 + dn) / 2)                  # the boundary on p's side of r
    exact = p == r64                                                           # x in {0, 1}, gamma 1, ...
    gap = np.abs(p - mid) / np.spacing(np.maximum(np.abs(p), np.abs(mid)))
    assert np.all(exact | (gap >= margin_ulps)), ("pow too close to an fp32 boundary", g, x64[~exact & (gap < margin_ulps)])
    return r


def tables(aug_row=None):
    """prep_u8_ex_kernel's lut[2][3][256] of one sample: image im (0: I, 1: I'), channel c, uint8 value x."""
    lut = np.empty((2, 3, 256), f32)
    x = np.arange(256)
    on = aug_row is not None and f32(aug_row[0]) != 0
    for im in range(2):
        if on:
            a = np.asarray(aug_row, f32)[1 + 5 * im:6 + 5 * im]
            p = pow_f32(x, a[0])
        for c in range(3):
            if on:
                v = (p * a[1]).astype(f32)
                v = (v * a[2 + c]).astype(f32)
                v = np.minimum(np.maximum(v, f32(0)), f32(255))
            else:
                v = x.astype(f32)
            lut[im, c] = ((v - MEAN[c]).astype(f32) / STD[c]).astype(f32)
    return lut


def _gray(l, px):
    """((l[0][r] + l[1][g]) + l[2][b]) / 3.0f over the [..., 3] uint8 pixels px."""
    return ((((l[0][px[..., 0]] + l[1][px[..., 1]]).astype(f32) + l[2][px[..., 2]]).astype(f32)) / f32(3)).astype(f32)


def origin_xy(pts1_row):
    return int(np.trunc(f32(pts1_row[0]))), int(np.trunc(f32(pts1_row[1])))     # (int)pts1: truncation


def prep_ex(I_u8, Ip_u8, pts1, aug, P):
    """udh_prep_inputs_u8_ex: I_gray [B,H,W,1], I_aug3 [B,H,W,3], I1, I2, I1_aug, I2_aug [B,P,P,1] and origin [B] int32.
    The patch outputs hold the window inside the image (the kernel writes only those elements)."""
    I_u8 = np.asarray(I_u8); Ip_u8 = np.asarray(Ip_u8)
    B, Hh, W, _ = I_u8.shape
    out = dict(I_gray=np.empty((B, Hh, W, 1), f32), I_aug3=np.empty((B, Hh, W, 3), f32),
               I1=np.empty((B, P, P, 1), f32), I2=np.empty((B, P, P, 1), f32), I1_aug=np.empty((B, P, P, 1), f32),
               I2_aug=np.empty((B, P, P, 1), f32), origin=np.empty(B, np.int32))
    plain = tables(None)
    for b in range(B):
        L = tables(None if aug is None else np.asarray(aug)[b])
        gI = _gray(L[0], I_u8[b])
        out["I_gray"][b, ..., 0] = gI
        for c in range(3):
            out["I_aug3"][b, ..., c] = L[0, c][I_u8[b, ..., c]]
        x0, y0 = origin_xy(pts1[b])
        out["origin"][b] = y0 * W + x0
        win = (slice(y0, y0 + P), slice(x0, x0 + P))
        out["I1_aug"][b, ..., 0] = gI[win]
        out["I2_aug"][b, ..., 0] = _gray(L[1], Ip_u8[b][win])
        out["I1"][b, ..., 0] = _gray(plain[0], I_u8[b][win])
        out["I2"][b, ..., 0] = _gray(plain[0], Ip_u8[b][win])
    return out


# ---------------------------------------------------------------------------- prep.cu
def normalise_u8(src_u8):
    """normalise_u8_kernel over the flat uint8 buffer (length a multiple of 4): float4 group i starts at channel
    (4i) % 3 and its four elements take channels c0, c0 + 1, c0 + 2, c0 (mod 3)."""
    flat = np.asarray(src_u8).reshape(-1)
    assert flat.size % 4 == 0
    q = flat.reshape(-1, 4).astype(f32)
    c0 = (np.arange(q.shape[0], dtype=np.int64) * 4) % 3
    ch = np.stack([c0, (c0 + 1) % 3, (c0 + 2) % 3, c0], 1)
    return (((q - MEAN[ch]).astype(f32)) / STD[ch]).astype(f32).reshape(-1)


def patches_u8(I_u8, Ip_u8, pts1, P):
    """patches_u8_kernel: I1, I2 [B,P,P] (gray_norm of each window pixel) and origin [B] int32."""
    B, Hh, W, _ = np.asarray(I_u8).shape
    plain = tables(None)[0]
    I1 = np.empty((B, P, P), f32); I2 = np.empty((B, P, P), f32); org = np.empty(B, np.int32)
    for b in range(B):
        x0, y0 = origin_xy(pts1[b])
        org[b] = y0 * W + x0
        I1[b] = _gray(plain, I_u8[b, y0:y0 + P, x0:x0 + P])
        I2[b] = _gray(plain, Ip_u8[b, y0:y0 + P, x0:x0 + P])
    return I1, I2, org
