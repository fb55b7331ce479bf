// cv2.warpPerspective(src, M, (dst_w, dst_h)) with its defaults (INTER_LINEAR, BORDER_CONSTANT, border value 0) on batched
// uint8 images of 1 or 3 channels, bit for bit (oracle/warp_perspective.py states the rules and how they were settled):
//   inverse   M is inverted in float64 by the 3x3 cofactor rule (zero matrix when the determinant is 0);
//   coords    per output pixel, in float64 without FMA, relative to its tile column xb (tiles of bw columns):
//             X0 = Mi0 xb + Mi1 y + Mi2 ...; W = W0 + Mi6 (x - xb); W = W ? 32 / W : 0;
//             X = round_half_even(clamp((X0 + Mi0 (x - xb)) W, INT_MIN, INT_MAX)) in 1/32 pixel (likewise Y);
//   sample    taps (X >> 5, Y >> 5) + {0,1}^2 (saturated to int16), 15-bit weights 32 (32 - fx)(32 - fy) ..., a tap outside
//             the source contributes 0, (sum + 2^14) >> 15.
// Laid out for bandwidth: each thread makes four consecutive output pixels of one item and stores them as 32-bit words
// (4 C bytes), so a warp writes 128 C contiguous bytes; the 4 C taps of a pixel are read through the read-only data cache,
// where neighbouring output pixels share them.  It does not reach HBM's bound (DESIGN section 5): the float64 coordinate
// arithmetic, one IEEE division per pixel, is part of the rounding contract.
// The sequence mosaic's blends (udh_mosaic_blend_u8 and udh_mosaic_multiband_u8, below) sample every frame with the same
// coordinate and tap helpers.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <vector>

#include "common.cuh"
#include "roi_warp.cuh"

namespace udh {

template <int C>
__device__ __forceinline__ void wp_pixel(const uint8_t* __restrict__ s, int h, int w, const double* mi, int x, int y, int bw,
                                         uint8_t* out) {
  int X, Y, v[C];
  wp_coords(mi, x, y, bw, X, Y);
  wp_sample<C>(s, h, w, X, Y, v);
#pragma unroll
  for (int c = 0; c < C; ++c) out[c] = (uint8_t)v[c];
}

template <int C>
__global__ void __launch_bounds__(256) warp_perspective_u8_kernel(const uint8_t* __restrict__ src, const double* __restrict__ M, int h,
                                                                  int w, uint8_t* __restrict__ dst, int dh, int dw, int bw) {
  __shared__ double mi[9];
  const int b = blockIdx.y;
  if (threadIdx.x == 0) cv_invert3(M + (int64_t)b * 9, mi);
  __syncthreads();
  const int npx = dh * dw;                                             // < 2^30: sides < 32767
  const int p0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (p0 >= npx) return;
  const uint8_t* s = src + (int64_t)b * h * w * C;
  uint8_t* d = dst + ((int64_t)b * npx + p0) * C;
  const int n = npx - p0 < 4 ? npx - p0 : 4;
  int y = p0 / dw, x = p0 - y * dw;
  alignas(4) uint8_t px[4 * C];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (k < n) wp_pixel<C>(s, h, w, mi, x, y, bw, px + k * C);
    if (++x == dw) { x = 0; ++y; }
  }
  if (n == 4 && (reinterpret_cast<uintptr_t>(d) & 3) == 0) {
#pragma unroll
    for (int k = 0; k < C; ++k) reinterpret_cast<uint32_t*>(d)[k] = reinterpret_cast<const uint32_t*>(px)[k];
  } else {
#pragma unroll
    for (int k = 0; k < 4 * C; ++k)
      if (k < n * C) d[k] = px[k];
  }
}

// ---- sequence mosaic: every frame warped onto one canvas and blended (the blend rule: oracle/mosaic.py) ---------------
struct MosaicFrame {
  double mi[9];                   // cv_invert3 of the frame's M (frame -> canvas), filled by invert_kernel
  const uint8_t* src;
  int h, w;
};

// Every frame's inverse into its table entry: fr[k].mi = cv_invert3(M_k).
template <class Frame>
__global__ void invert_kernel(const double* __restrict__ M, Frame* fr, int n) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) cv_invert3(M + (int64_t)k * 9, fr[k].mi);
}

// A frame's blend mask on the canvas (udh_mosaic_seam_masks_u8's output): 0 / 255 bytes on its ROI rectangle.  An empty
// rectangle (rw = 0) masks the whole frame out.
struct SeamMask {
  const uint8_t* m;
  int rx, ry, rw, rh;
};

__device__ __forceinline__ bool seam_mask_on(const SeamMask* __restrict__ sm, int x, int y) {
  const int lx = x - __ldg(&sm->rx), ly = y - __ldg(&sm->ry), rw = __ldg(&sm->rw);
  if ((unsigned)lx >= (unsigned)rw || (unsigned)ly >= (unsigned)__ldg(&sm->rh)) return false;
  const uint8_t* m = reinterpret_cast<const uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&sm->m)));
  return __ldg(m + (int64_t)ly * rw + lx) != 0;
}

// Exposure compensation's apply, cv2.multiply(uint8, double): saturate_u8(rint(v g)) in float64, ties to even.
__device__ __forceinline__ int ex_apply(int v, double g) {
  return min(max(__double2int_rn(__dmul_rn((double)v, g)), 0), 255);
}

// Block exposure compensation's apply, cv2.multiply(uint8, float32 map, CV_8U): saturate_u8(rint(float32(v) g)) in float32.
__device__ __forceinline__ int ex_apply_f(int v, float g) {
  return min(max(__float2int_rn(__fmul_rn((float)v, g)), 0), 255);
}

// A frame's gain map with its ROI rectangle (rx, ry, rw, rh) on the canvas.
struct GainMapDev {
  udh_gain_map m;
  int rx, ry, rw, rh;
};

// The gain map's bilinear resize at ROI pixel (lx, ly): g[c] for c < 3 (the one gain repeated when the map has 1 channel).
// The row pass, then the column pass, every product and sum rounded to float32 (oracle/exposure_blocks.resize_map).
__device__ __forceinline__ void gm_gains(const GainMapDev* __restrict__ G, int lx, int ly, float* g) {
  const float* mp = reinterpret_cast<const float*>(__ldg(reinterpret_cast<const unsigned long long*>(&G->m.map)));
  const udh_map_tap* ct = reinterpret_cast<const udh_map_tap*>(__ldg(reinterpret_cast<const unsigned long long*>(&G->m.cols)));
  const udh_map_tap* rt = reinterpret_cast<const udh_map_tap*>(__ldg(reinterpret_cast<const unsigned long long*>(&G->m.rows)));
  const int bpx = __ldg(&G->m.bpx), ch = __ldg(&G->m.channels);
  const int cs0 = __ldg(&ct[lx].s0), cs1 = __ldg(&ct[lx].s1), rs0 = __ldg(&rt[ly].s0), rs1 = __ldg(&rt[ly].s1);
  const float ca0 = __ldg(&ct[lx].a0), ca1 = __ldg(&ct[lx].a1), ra0 = __ldg(&rt[ly].a0), ra1 = __ldg(&rt[ly].a1);
  for (int c = 0; c < 3; ++c) {
    if (c >= ch) {
      g[c] = g[0];
      continue;
    }
    const float* r0 = mp + ((int64_t)rs0 * bpx) * ch + c;
    const float* r1 = mp + ((int64_t)rs1 * bpx) * ch + c;
    const float h0 = __fadd_rn(__fmul_rn(__ldg(r0 + cs0 * ch), ca0), __fmul_rn(__ldg(r0 + cs1 * ch), ca1));
    const float h1 = __fadd_rn(__fmul_rn(__ldg(r1 + cs0 * ch), ca0), __fmul_rn(__ldg(r1 + cs1 * ch), ca1));
    g[c] = __fadd_rn(__fmul_rn(h0, ra0), __fmul_rn(h1, ra1));
  }
}

// Gather form: one CTA per UDH_MOSAIC_TILE_H x UDH_MOSAIC_TILE_W canvas tile, each thread four consecutive pixels of one
// row.  The thread walks the tile's candidate frames, adds wt * v and wt of every frame valid at its pixels into 64-bit
// registers and stores the pixels once: no atomics, no accumulation buffer.  Integer sums: the result does not depend on
// the frames' order.  GAIN: each frame's value is first compensated, ex_apply(v, gains[f][c]) (channel 0's gain when C = 1).
// MASK: a frame counts only where its blend mask smask[f] is set as well.  MAP: each frame's value is compensated by its
// gain map at the pixel's ROI coordinates (gm_gains).  The optional tables come last, so the plain blend's parameters keep
// their offsets and its code is the feathered blend's own.
template <int C, bool GAIN, bool MASK, bool MAP>
__global__ void __launch_bounds__(256) mosaic_blend_u8_kernel(const MosaicFrame* __restrict__ fr, int n, const int32_t* __restrict__ tile_ptr,
                                                              const int32_t* __restrict__ tile_frames, int dh, int dw, int bw,
                                                              int feather32, uint8_t* __restrict__ dst, uint8_t* __restrict__ mask,
                                                              const double* __restrict__ gains, const SeamMask* __restrict__ smask,
                                                              const GainMapDev* __restrict__ gmap) {
  const int y = blockIdx.y * UDH_MOSAIC_TILE_H + threadIdx.x / (UDH_MOSAIC_TILE_W / 4);
  const int x0 = blockIdx.x * UDH_MOSAIC_TILE_W + threadIdx.x % (UDH_MOSAIC_TILE_W / 4) * 4;
  if (y >= dh || x0 >= dw) return;
  const int np = dw - x0 < 4 ? dw - x0 : 4;
  const int tile = blockIdx.y * gridDim.x + blockIdx.x;
  uint64_t S[4][C], D[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    D[k] = 0;
#pragma unroll
    for (int c = 0; c < C; ++c) S[k][c] = 0;
  }
  const int j1 = __ldg(tile_ptr + tile + 1);
  for (int j = __ldg(tile_ptr + tile); j < j1; ++j) {
    const int f = __ldg(tile_frames + j);
    if ((unsigned)f >= (unsigned)n) continue;
    const MosaicFrame* F = fr + f;
    double mi[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) mi[k] = __ldg(F->mi + k);
    const uint8_t* s = reinterpret_cast<const uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&F->src)));
    const int h = __ldg(&F->h), w = __ldg(&F->w);
    const int xm = 32 * (w - 1), ym = 32 * (h - 1);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (k >= np) break;
      int X, Y;
      const double Wd = wp_coords(mi, x0 + k, y, bw, X, Y);
      if (Wd != 0.0 && X >= 0 && X <= xm && Y >= 0 && Y <= ym && (!MASK || seam_mask_on(smask + f, x0 + k, y))) {
        const int wt = 1 + min(min(min(X, xm - X), min(Y, ym - Y)), feather32);
        int v[C];
        wp_sample<C>(s, h, w, X, Y, v);
        if (GAIN) {
#pragma unroll
          for (int c = 0; c < C; ++c) v[c] = ex_apply(v[c], __ldg(gains + 3 * f + c));
        }
        if (MAP) {
          const GainMapDev* G = gmap + f;
          float g[3];
          gm_gains(G, min(max(x0 + k - __ldg(&G->rx), 0), __ldg(&G->rw) - 1), min(max(y - __ldg(&G->ry), 0), __ldg(&G->rh) - 1), g);
#pragma unroll
          for (int c = 0; c < C; ++c) v[c] = ex_apply_f(v[c], g[c]);
        }
#pragma unroll
        for (int c = 0; c < C; ++c) S[k][c] += (uint64_t)(wt * v[c]);
        D[k] += (uint64_t)wt;
      }
    }
  }
  alignas(4) uint8_t px[4 * C];
  alignas(4) uint8_t mk[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    mk[k] = D[k] ? 255 : 0;
#pragma unroll
    for (int c = 0; c < C; ++c) px[k * C + c] = D[k] ? (uint8_t)((S[k][c] + (D[k] >> 1)) / D[k]) : 0;
  }
  const int64_t p0 = (int64_t)y * dw + x0;
  uint8_t* d = dst + p0 * C;
  uint8_t* m = mask + p0;
  if (np == 4 && (reinterpret_cast<uintptr_t>(d) & 3) == 0) {
#pragma unroll
    for (int k = 0; k < C; ++k) reinterpret_cast<uint32_t*>(d)[k] = reinterpret_cast<const uint32_t*>(px)[k];
  } else {
#pragma unroll
    for (int k = 0; k < 4 * C; ++k)
      if (k < np * C) d[k] = px[k];
  }
  if (np == 4 && (reinterpret_cast<uintptr_t>(m) & 3) == 0) {
    *reinterpret_cast<uint32_t*>(m) = *reinterpret_cast<const uint32_t*>(mk);
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k < np) m[k] = mk[k];
  }
}

// ---- multi-band blend: cv2.detail_MultiBandBlender with CV_16S weights (the rule: oracle/multiband.py) ----------------
// Per frame k, its fed rectangle (ROI grown by the gap, aligned to 2^B) holds the image pyramid G_i (uchar4, RGB + pad)
// and the weight pyramid W_i (int16) in two pools; the canvas pyramid keeps (acc, wacc) as short4 per pixel, and the
// collapsed levels R_i (i >= 1) as short4 in a second pyramid, so acc and wacc survive the blend.
constexpr int MB_MAX_BANDS = 10;

struct MultibandFrame : RoiFrame {
  int x0, y0, pw, ph;              // the fed rectangle at level 0 (canvas coordinates; multiples of 2^B)
  int64_t off[MB_MAX_BANDS + 1];   // element offset of level i in the G and W pools
  const uint8_t* bmask;            // null, or the frame's blend mask on its ROI (rh x rw, 0 / 255): the weight's mask
};

// BORDER_REFLECT (fedcba|abcdef|fedcba) for any n >= 1, folding as often as needed.
__device__ __forceinline__ int mb_reflect(int i, int n) {
  if (n == 1) return 0;
  int p = i % (2 * n);
  if (p < 0) p += 2 * n;
  return p < n ? p : 2 * n - 1 - p;
}

// cv2.pyrUp's taps along one axis at output o of a source of n: -1 reads 1 (reflect-101), n reads n - 1 (reflect).
__device__ __forceinline__ void mb_up_taps(int o, int n, int* t, int* wt) {
  const int j = o >> 1;
  if (o & 1) {
    t[0] = j; t[1] = j + 1; t[2] = j + 1;
    wt[0] = 4; wt[1] = 4; wt[2] = 0;
  } else {
    t[0] = j - 1; t[1] = j; t[2] = j + 1;
    wt[0] = 1; wt[1] = 6; wt[2] = 1;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) t[k] = t[k] < 0 ? min(1, n - 1) : min(t[k], n - 1);
}

__device__ __forceinline__ int mb_sat16(int v) { return min(max(v, -32768), 32767); }

// Level 0 of every frame: the ROI warp bordered with BORDER_REFLECT, and the 0 / 256 weight with a constant 0 border.
// gains (null: none) [n][3]: the ROI warp is exposure-compensated first, ex_apply(v, gains[k][c]), as cv2's stitcher
// applies its compensator to the whole warped image before it feeds the blender.  A frame with a blend mask (bmask) takes
// its weight from that mask instead of the warp's validity: mask + 1 where the mask is nonzero, cv2's CV_16S feed (255 ->
// 256; a graded seam-scale mask weighs 2 .. 255 along its seams).
// MAP: the ROI warp is compensated by the frame's gain map at each ROI pixel instead (gm_gains, ex_apply_f).
template <bool MAP>
__global__ void __launch_bounds__(256) multiband_base_kernel(const MultibandFrame* __restrict__ fr, const double* __restrict__ M,
                                                             const double* __restrict__ gains, const GainMapDev* __restrict__ gmap,
                                                             uchar4* __restrict__ G, int16_t* __restrict__ Wt) {
  __shared__ double mi[9];
  const int k = blockIdx.y;
  if (threadIdx.x == 0) cv_invert3(M + (int64_t)k * 9, mi);
  __syncthreads();
  const MultibandFrame* F = fr + k;
  const uint8_t* s = reinterpret_cast<const uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&F->src)));
  const int h = __ldg(&F->h), w = __ldg(&F->w), rx = __ldg(&F->rx), ry = __ldg(&F->ry), rw = __ldg(&F->rw), rh = __ldg(&F->rh);
  const int bw = __ldg(&F->bw), ox = __ldg(&F->x0) - rx, oy = __ldg(&F->y0) - ry, pw = __ldg(&F->pw);
  const int npx = pw * __ldg(&F->ph);                                 // < 2^31: padded sides < 32767 + 1024
  const int64_t off = __ldg(&F->off[0]);
  const uint8_t* bm = reinterpret_cast<const uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&F->bmask)));
  double g[3];
  if (!MAP && gains) {
#pragma unroll
    for (int c = 0; c < 3; ++c) g[c] = __ldg(gains + 3 * k + c);
  }
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < npx; e += gridDim.x * blockDim.x) {
    const int y = e / pw, x = e - y * pw;
    const int ix = x + ox, iy = y + oy;
    const int sx = mb_reflect(ix, rw), sy = mb_reflect(iy, rh);
    int v[3];
    const bool valid = mb_roi_warp(s, h, w, mi, sx, sy, bw, v) && ix == sx && iy == sy;
    int wt = valid ? 256 : 0;
    if (bm) {
      const int b = ix == sx && iy == sy ? __ldg(bm + (int64_t)sy * rw + sx) : 0;
      wt = b ? b + 1 : 0;
    }
    Wt[off + e] = (int16_t)wt;
    if (MAP) {
      float gf[3];
      gm_gains(gmap + k, sx, sy, gf);
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = ex_apply_f(v[c], gf[c]);
    } else if (gains) {
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = ex_apply(v[c], g[c]);
    }
    G[off + e] = make_uchar4((unsigned char)v[0], (unsigned char)v[1], (unsigned char)v[2], 0);
  }
}

// Level lvl -> lvl + 1 of every frame's G and W: cv2.pyrDown (taps 1 4 6 4 1, BORDER_REFLECT_101, (sum + 128) >> 8).
__global__ void __launch_bounds__(256) multiband_down_kernel(const MultibandFrame* __restrict__ fr, uchar4* __restrict__ G,
                                                             int16_t* __restrict__ Wt, int lvl) {
  const MultibandFrame* F = fr + blockIdx.y;
  const int sw = __ldg(&F->pw) >> lvl, sh = __ldg(&F->ph) >> lvl, dw = sw >> 1, npx = dw * (sh >> 1);
  const int64_t si = __ldg(&F->off[lvl]), di = __ldg(&F->off[lvl + 1]);
  const int kw[5] = {1, 4, 6, 4, 1};
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < npx; e += gridDim.x * blockDim.x) {
    const int y = e / dw, x = e - y * dw;
    int tx[5];
#pragma unroll
    for (int j = 0; j < 5; ++j) tx[j] = reflect101(2 * x + j - 2, sw);
    int a0 = 0, a1 = 0, a2 = 0, aw = 0;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const int64_t row = si + (int64_t)reflect101(2 * y + i - 2, sh) * sw;
      int r0 = 0, r1 = 0, r2 = 0, rw = 0;
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        const uchar4 g = G[row + tx[j]];
        r0 += kw[j] * g.x; r1 += kw[j] * g.y; r2 += kw[j] * g.z;
        rw += kw[j] * Wt[row + tx[j]];
      }
      a0 += kw[i] * r0; a1 += kw[i] * r1; a2 += kw[i] * r2; aw += kw[i] * rw;
    }
    G[di + e] = make_uchar4((unsigned char)((a0 + 128) >> 8), (unsigned char)((a1 + 128) >> 8), (unsigned char)((a2 + 128) >> 8), 0);
    Wt[di + e] = (int16_t)mb_sat16((aw + 128) >> 8);
  }
}

// Gather form, level lvl of the canvas pyramid: one thread per pixel of a MB_TILE_W x MB_TILE_H tile.  The CTA collects the
// frames whose rectangle at this level meets its tile (256 at a time), and each thread sums (L W) >> 8 and W of every such
// frame in int32 and stores them once, truncated to int16: the same bytes as cv2's wrapping int16 adds, in any frame order.
// L = G_lvl - pyrUp(G_lvl+1), formed on the fly (G_B at the top).
constexpr int MB_TILE_W = 32, MB_TILE_H = 8;

__global__ void __launch_bounds__(256) multiband_accumulate_kernel(const MultibandFrame* __restrict__ fr, int n,
                                                                   const uchar4* __restrict__ G, const int16_t* __restrict__ Wt,
                                                                   int lvl, int top, int cw, int ch, short4* __restrict__ acc) {
  __shared__ int cand[256];
  __shared__ int ncand;
  const int tx0 = blockIdx.x * MB_TILE_W, ty0 = blockIdx.y * MB_TILE_H;
  const int x = tx0 + threadIdx.x % MB_TILE_W, y = ty0 + threadIdx.x / MB_TILE_W;
  int a0 = 0, a1 = 0, a2 = 0, aw = 0;
  for (int c0 = 0; c0 < n; c0 += 256) {
    if (threadIdx.x == 0) ncand = 0;
    __syncthreads();
    const int k = c0 + threadIdx.x;
    if (k < n) {
      const MultibandFrame* F = fr + k;
      const int fx0 = __ldg(&F->x0) >> lvl, fy0 = __ldg(&F->y0) >> lvl;
      const int fx1 = fx0 + (__ldg(&F->pw) >> lvl), fy1 = fy0 + (__ldg(&F->ph) >> lvl);
      if (fx0 < tx0 + MB_TILE_W && fx1 > tx0 && fy0 < ty0 + MB_TILE_H && fy1 > ty0) cand[atomicAdd(&ncand, 1)] = k;
    }
    __syncthreads();
    const int nc = ncand;
    for (int j = 0; j < nc; ++j) {
      const MultibandFrame* F = fr + cand[j];
      const int fw = __ldg(&F->pw) >> lvl, fh = __ldg(&F->ph) >> lvl;
      const int lx = x - (__ldg(&F->x0) >> lvl), ly = y - (__ldg(&F->y0) >> lvl);
      if ((unsigned)lx >= (unsigned)fw || (unsigned)ly >= (unsigned)fh) continue;
      const int64_t p = __ldg(&F->off[lvl]) + (int64_t)ly * fw + lx;
      const int wt = Wt[p];
      if (wt == 0) continue;                                            // adds 0 to both sums
      const uchar4 g = G[p];
      int l0 = g.x, l1 = g.y, l2 = g.z;
      if (!top) {
        const int uw = fw >> 1, uh = fh >> 1;
        const int64_t u0 = __ldg(&F->off[lvl + 1]);
        int txs[3], wxs[3], tys[3], wys[3];
        mb_up_taps(lx, uw, txs, wxs);
        mb_up_taps(ly, uh, tys, wys);
        int s0 = 0, s1 = 0, s2 = 0;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          if (wys[i] == 0) continue;
          int r0 = 0, r1 = 0, r2 = 0;
#pragma unroll
          for (int q = 0; q < 3; ++q) {
            if (wxs[q] == 0) continue;
            const uchar4 u = G[u0 + (int64_t)tys[i] * uw + txs[q]];
            r0 += wxs[q] * u.x; r1 += wxs[q] * u.y; r2 += wxs[q] * u.z;
          }
          s0 += wys[i] * r0; s1 += wys[i] * r1; s2 += wys[i] * r2;
        }
        l0 -= (s0 + 32) >> 6; l1 -= (s1 + 32) >> 6; l2 -= (s2 + 32) >> 6;
      }
      a0 += (l0 * wt) >> 8; a1 += (l1 * wt) >> 8; a2 += (l2 * wt) >> 8;
      aw += wt;
    }
    __syncthreads();
  }
  if (x < cw && y < ch) acc[(int64_t)y * cw + x] = make_short4((short)a0, (short)a1, (short)a2, (short)aw);
}

// cv2's normalisation: (int16)((acc << 8) / (wacc + 1)), truncating.  cv2 divides by zero where wacc = -1; this writes 0.
__device__ __forceinline__ int mb_norm(int a, int wacc) {
  const int d = wacc + 1;
  return d ? (short)((a * 256) / d) : 0;
}

// Level lvl of the collapse: R = sat16(pyrUp(R_lvl+1) + N) (N alone at the top).  FINAL (level 0) writes the cropped
// uint8 RGB mosaic and the 0 / 255 mask (wacc > 0) instead of R.
template <bool FINAL>
__global__ void __launch_bounds__(256) multiband_collapse_kernel(const short4* __restrict__ acc, const short4* __restrict__ up,
                                                                 int cw, int ch, short4* __restrict__ R, int dh, int dw,
                                                                 uint8_t* __restrict__ dst, uint8_t* __restrict__ mask) {
  const int ow = FINAL ? dw : cw, npx = FINAL ? dh * dw : cw * ch;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < npx; e += gridDim.x * blockDim.x) {
    const int y = e / ow, x = e - y * ow;
    const short4 a = acc[(int64_t)y * cw + x];
    int v0 = mb_norm(a.x, a.w), v1 = mb_norm(a.y, a.w), v2 = mb_norm(a.z, a.w);
    if (up) {
      const int uw = cw >> 1, uh = ch >> 1;
      int txs[3], wxs[3], tys[3], wys[3];
      mb_up_taps(x, uw, txs, wxs);
      mb_up_taps(y, uh, tys, wys);
      int s0 = 0, s1 = 0, s2 = 0;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        if (wys[i] == 0) continue;
        int r0 = 0, r1 = 0, r2 = 0;
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          if (wxs[q] == 0) continue;
          const short4 u = up[(int64_t)tys[i] * uw + txs[q]];
          r0 += wxs[q] * u.x; r1 += wxs[q] * u.y; r2 += wxs[q] * u.z;
        }
        s0 += wys[i] * r0; s1 += wys[i] * r1; s2 += wys[i] * r2;
      }
      v0 = mb_sat16(mb_sat16((s0 + 32) >> 6) + v0);
      v1 = mb_sat16(mb_sat16((s1 + 32) >> 6) + v1);
      v2 = mb_sat16(mb_sat16((s2 + 32) >> 6) + v2);
    }
    if (FINAL) {
      const bool m = a.w > 0;
      uint8_t* d = dst + ((int64_t)y * dw + x) * 3;
      d[0] = m ? (uint8_t)min(max(v0, 0), 255) : 0;
      d[1] = m ? (uint8_t)min(max(v1, 0), 255) : 0;
      d[2] = m ? (uint8_t)min(max(v2, 0), 255) : 0;
      mask[(int64_t)y * dw + x] = m ? 255 : 0;
    } else {
      R[(int64_t)y * cw + x] = make_short4((short)v0, (short)v1, (short)v2, 0);
    }
  }
}

// The host's plan of one multi-band call: bands, padded canvas, frame table and workspace layout.
struct MultibandPlan {
  int B, Hp, Wp, max_px[MB_MAX_BANDS + 1];
  int64_t E;                                                          // elements per pool
  size_t off_g, off_w, off_acc[MB_MAX_BANDS + 1], off_r[MB_MAX_BANDS + 1], total;
  std::vector<MultibandFrame> fr;
};

// rois [n,4] (x_lo, y_lo, x_hi, y_hi) -> plan (frames and sizes may be null: the frame fields are left unset).  0 or an error.
static int mb_plan(const uint8_t* const* frames, const int32_t* rois, const int32_t* sizes, int n, int Hc, int Wc, int bands,
                   MultibandPlan& p) {
  UDH_REQUIRE(n >= 1 && n <= 65535 && Hc >= 1 && Wc >= 1 && Hc < 32767 && Wc < 32767,
              "udh_mosaic_multiband_u8: bad dimensions (n %d, canvas %dx%d)", n, Hc, Wc);
  UDH_REQUIRE(bands >= 0 && bands <= MB_MAX_BANDS, "udh_mosaic_multiband_u8: bands must be in [0, %d] (got %d)", MB_MAX_BANDS, bands);
  UDH_REQUIRE(rois, "udh_mosaic_multiband_u8: null rois");
  // cv2's band count: min(B, ceil(log(max side) / log 2)) in double
  const int lg = (int)std::ceil(std::log((double)(Hc > Wc ? Hc : Wc)) / std::log(2.0));
  p.B = bands < lg ? bands : lg;
  const int a = 1 << p.B, gap = 3 << p.B;
  p.Hp = Hc + (a - Hc % a) % a;
  p.Wp = Wc + (a - Wc % a) % a;
  p.fr.assign((size_t)n, MultibandFrame{});
  for (int i = 0; i <= MB_MAX_BANDS; ++i) p.max_px[i] = 0;
  int64_t E = 0;
  for (int k = 0; k < n; ++k) {
    MultibandFrame& F = p.fr[k];
    const int rc = roi_frame(frames, sizes, rois, k, Hc, Wc, F, "udh_mosaic_multiband_u8");
    if (rc != UDH_OK) return rc;
    // cv2's tl_new / br_new: grow by the gap, clip, align to 2^B, shift back inside the padded canvas
    int x0 = F.rx - gap > 0 ? F.rx - gap : 0, y0 = F.ry - gap > 0 ? F.ry - gap : 0;
    int x1 = F.rx + F.rw + gap < p.Wp ? F.rx + F.rw + gap : p.Wp, y1 = F.ry + F.rh + gap < p.Hp ? F.ry + F.rh + gap : p.Hp;
    x0 = (x0 >> p.B) << p.B;
    y0 = (y0 >> p.B) << p.B;
    x1 = x0 + (x1 - x0) + (a - (x1 - x0) % a) % a;
    y1 = y0 + (y1 - y0) + (a - (y1 - y0) % a) % a;
    const int dx = x1 - p.Wp > 0 ? x1 - p.Wp : 0, dy = y1 - p.Hp > 0 ? y1 - p.Hp : 0;
    F.x0 = x0 - dx; F.y0 = y0 - dy; F.pw = x1 - x0; F.ph = y1 - y0;
    for (int i = 0; i <= p.B; ++i) {
      const int px = (F.pw >> i) * (F.ph >> i);
      F.off[i] = E;
      E += px;
      if (px > p.max_px[i]) p.max_px[i] = px;
    }
  }
  p.E = E;
  size_t o = mb_align((size_t)n * sizeof(MultibandFrame));
  p.off_g = o;
  o = mb_align(o + (size_t)E * sizeof(uchar4));
  p.off_w = o;
  o = mb_align(o + (size_t)E * sizeof(int16_t));
  for (int i = 0; i <= p.B; ++i) {
    p.off_acc[i] = o;
    o = mb_align(o + (size_t)(p.Hp >> i) * (size_t)(p.Wp >> i) * sizeof(short4));
  }
  p.off_r[0] = 0;
  for (int i = 1; i <= p.B; ++i) {
    p.off_r[i] = o;
    o = mb_align(o + (size_t)(p.Hp >> i) * (size_t)(p.Wp >> i) * sizeof(short4));
  }
  p.total = o;
  return UDH_OK;
}

// ---- exposure compensation: per-pair statistics of the ROI warps (cv2.detail's gain compensators; oracle/exposure.py) ----
// For every listed pair i <= j of frames whose ROIs intersect, over the canvas pixels where both ROI warps are valid:
// the count, each frame's channel sums and, with norms, each frame's sum of sqrt(r^2 + g^2 + b^2) (cv2's norm(Vec3b)).
// Such a norm is 0 or a multiple of 2^-52 below 2^9, so q = norm 2^52 is an integer below 2^61; it is summed exactly as
// three 21-bit limbs (each limb's sum stays below 2^52 for up to 2^31 pixels), and the host rounds the total once.
struct ExposureFrame : RoiFrame {
  double mi[9];                    // cv_invert3 of M'_k (frame -> its ROI)
};

constexpr int EX_TILE_W = 32, EX_TILE_H = 64, EX_CHUNK = 8, EX_PAIRS = EX_CHUNK * EX_CHUNK;

// The frames whose ROI meets the CTA's EX_TILE_W x EX_TILE_H tile at (tx0, ty0), in ascending frame order, into cand: per
// 256 frames, each warp's ballot, ranked by the warps before it.  Returns their count.
template <class Frame>
__device__ __forceinline__ int ex_candidates(const Frame* __restrict__ fr, int n, int tx0, int ty0, int* cand, int* wcount) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int nc = 0;
  for (int c0 = 0; c0 < n; c0 += blockDim.x) {
    const int k = c0 + threadIdx.x;
    bool hit = false;
    if (k < n) {
      const Frame* F = fr + k;
      const int rx = __ldg(&F->rx), ry = __ldg(&F->ry);
      hit = rx < tx0 + EX_TILE_W && rx + __ldg(&F->rw) > tx0 && ry < ty0 + EX_TILE_H && ry + __ldg(&F->rh) > ty0;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) wcount[warp] = __popc(bal);
    __syncthreads();
    int base = nc, tot = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      base += q < warp ? wcount[q] : 0;
      tot += wcount[q];
    }
    if (hit) cand[base + __popc(bal & ((1u << lane) - 1u))] = k;
    nc += tot;
    __syncthreads();                                                  // wcount is rewritten next round
  }
  return nc;
}

// The index of pair (i, j) in the CSR pair list (row i, ascending j), or -1 when the pair is not listed.
__device__ __forceinline__ int ex_pair(const int32_t* __restrict__ pair_ptr, const int32_t* __restrict__ pair_j, int i, int j) {
  int lo = __ldg(pair_ptr + i), hi = __ldg(pair_ptr + i + 1);
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(pair_j + mid) < j) lo = mid + 1; else hi = mid;
  }
  return lo < __ldg(pair_ptr + i + 1) && __ldg(pair_j + lo) == j ? lo : -1;
}

// Gather form: one CTA per EX_TILE_W x EX_TILE_H canvas tile, each warp one row of 32 pixels at a time.  The CTA lists
// the frames whose ROI meets its tile in ascending frame order and takes them EX_CHUNK at a time, two chunks A <= B per
// round.  Per row each lane stores the compensated ROI-warp value and validity of every frame of A and B at its pixel in
// shared memory; then, for every listed pair of the round (looked up in the pair CSR), the warp sums its lanes' terms
// with __reduce_add_sync and adds them to the CTA's 64-bit sums, which are added to the pair's global sums once per
// round.  The ascending list puts the pair's lower frame i first in every slot (chunk A <= B, and a <= b within one
// chunk), so frame i's sums always go to i's fields.  Every sum is an integer, so the result does not depend on the
// frames' order, the tiling or the run.
// hist [feeds][n][3]: frame k's value is ex_apply'd with hist[0][k][c], then hist[1][k][c], ... (feed `feeds` of cv2's loop).
__global__ void __launch_bounds__(256) exposure_stats_kernel(const ExposureFrame* __restrict__ fr, int n,
                                                             const int32_t* __restrict__ pair_ptr,
                                                             const int32_t* __restrict__ pair_j, const double* __restrict__ hist,
                                                             int feeds, int norms, unsigned long long* __restrict__ stats) {
  __shared__ int cand[UDH_EXPOSURE_MAX_FRAMES];
  __shared__ int wcount[8];
  __shared__ uchar4 val[2 * EX_CHUNK][256];                             // .w: valid
  __shared__ int pidx[EX_PAIRS];
  __shared__ unsigned long long acc[EX_PAIRS][UDH_EXPOSURE_STATS];
  const int tx0 = blockIdx.x * EX_TILE_W, ty0 = blockIdx.y * EX_TILE_H;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nc = ex_candidates(fr, n, tx0, ty0, cand, wcount);
  const int nch = (nc + EX_CHUNK - 1) / EX_CHUNK;
  for (int A = 0; A < nch; ++A) {
    for (int B = A; B < nch; ++B) {
      // the round's pairs: slot t = a EX_CHUNK + b pairs frame a of chunk A with frame b of chunk B (a <= b when A = B)
      if (threadIdx.x < EX_PAIRS) {
        const int a = threadIdx.x / EX_CHUNK, b = threadIdx.x % EX_CHUNK, ka = A * EX_CHUNK + a, kb = B * EX_CHUNK + b;
        int p = -1;
        if (ka < nc && kb < nc && (A != B || a <= b)) p = ex_pair(pair_ptr, pair_j, cand[ka], cand[kb]);   // i <= j: the list ascends
        pidx[threadIdx.x] = p;
      }
      for (int e = threadIdx.x; e < EX_PAIRS * UDH_EXPOSURE_STATS; e += blockDim.x) (&acc[0][0])[e] = 0;
      __syncthreads();
      const int nA = min(EX_CHUNK, nc - A * EX_CHUNK), nB = A == B ? 0 : min(EX_CHUNK, nc - B * EX_CHUNK);
      for (int r = warp; r < EX_TILE_H; r += 8) {
        const int x = tx0 + lane, y = ty0 + r;
        for (int q = 0; q < nA + nB; ++q) {
          const int k = cand[q < nA ? A * EX_CHUNK + q : B * EX_CHUNK + q - nA];
          const ExposureFrame* F = fr + k;
          const int sx = x - __ldg(&F->rx), sy = y - __ldg(&F->ry);
          int v[3] = {0, 0, 0};
          bool ok = false;
          if ((unsigned)sx < (unsigned)__ldg(&F->rw) && (unsigned)sy < (unsigned)__ldg(&F->rh)) {
            double mi[9];
#pragma unroll
            for (int t = 0; t < 9; ++t) mi[t] = __ldg(F->mi + t);
            const uint8_t* s = reinterpret_cast<const uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&F->src)));
            ok = mb_roi_warp(s, __ldg(&F->h), __ldg(&F->w), mi, sx, sy, __ldg(&F->bw), v);
            for (int f = 0; f < feeds; ++f) {
#pragma unroll
              for (int c = 0; c < 3; ++c) v[c] = ex_apply(v[c], __ldg(hist + ((int64_t)f * n + k) * 3 + c));
            }
          }
          val[q < nA ? q : EX_CHUNK + q - nA][threadIdx.x] = make_uchar4(v[0], v[1], v[2], ok);
        }
        __syncwarp();
        for (int t = 0; t < EX_PAIRS; ++t) {
          const int p = pidx[t];
          if (p < 0) continue;
          const int a = t / EX_CHUNK, b = t % EX_CHUNK;
          const uchar4 u = val[a][threadIdx.x], w = val[A == B ? b : EX_CHUNK + b][threadIdx.x];
          const bool both = u.w && w.w;
          if (!__any_sync(0xffffffffu, both)) continue;
          const unsigned m = both ? 1u : 0u;
          unsigned sum[UDH_EXPOSURE_STATS] = {};
          sum[0] = m;
          sum[1] = m * u.x; sum[2] = m * u.y; sum[3] = m * u.z;
          sum[4] = m * w.x; sum[5] = m * w.y; sum[6] = m * w.z;
          if (norms) {
            const uint64_t qu = __double2ull_rn(__dmul_rn(__dsqrt_rn((double)(u.x * u.x + u.y * u.y + u.z * u.z)), 0x1p52)) * m;
            const uint64_t qw = __double2ull_rn(__dmul_rn(__dsqrt_rn((double)(w.x * w.x + w.y * w.y + w.z * w.z)), 0x1p52)) * m;
#pragma unroll
            for (int l = 0; l < 3; ++l) {
              sum[7 + l] = (unsigned)(qu >> (21 * l)) & 0x1fffffu;
              sum[10 + l] = (unsigned)(qw >> (21 * l)) & 0x1fffffu;
            }
          }
#pragma unroll
          for (int q = 0; q < UDH_EXPOSURE_STATS; ++q) {
            if (q >= 7 && !norms) break;
            const unsigned tot = __reduce_add_sync(0xffffffffu, sum[q]);   // < 2^26: 32 lanes of < 2^21
            if (lane == 0 && tot) atomicAdd(&acc[t][q], (unsigned long long)tot);
          }
        }
        __syncwarp();
      }
      __syncthreads();
      for (int e = threadIdx.x; e < EX_PAIRS * UDH_EXPOSURE_STATS; e += blockDim.x) {
        const int t = e / UDH_EXPOSURE_STATS, q = e % UDH_EXPOSURE_STATS, p = pidx[t];
        const unsigned long long v = acc[t][q];
        if (p >= 0 && v) atomicAdd(stats + (int64_t)p * UDH_EXPOSURE_STATS + q, v);
      }
      __syncthreads();
    }
  }
}

// ---- block exposure compensation (cv2.detail's block compensators; oracle/exposure_blocks.py) ----------------------------
// The statistics of every block pair, in one pass over the canvas laid out as exposure_stats_kernel: the CTA's frames in
// ascending order, two chunks per round, each frame's compensated value, validity and block (bx, by) per row in shared
// memory.  A listed frame pair's block pair at a pixel names one cell of the pair's merged block grid (udh.h), so each
// warp groups its lanes by cell (__match_any_sync), sums each group's terms with __reduce_add_sync and its leader adds
// them to the cell's global sums.  Every sum is an integer: the result does not depend on the order or the run.
struct ExposureBlockFrame : RoiFrame {
  double mi[9];                    // cv_invert3 of M'_k (frame -> its ROI)
  int bkw, bkh, bpx;               // the blocks' width and height, blocks per row
  int64_t boff;                    // the frame's first block
};

__global__ void __launch_bounds__(256) gainblock_stats_kernel(const ExposureBlockFrame* __restrict__ fr, int n,
                                                                   const int32_t* __restrict__ pair_ptr,
                                                                   const int32_t* __restrict__ pair_j,
                                                                   const int64_t* __restrict__ cell_off,
                                                                   const int32_t* __restrict__ cell_nx, const double* __restrict__ hist,
                                                                   int64_t nblocks, int feeds, int norms,
                                                                   unsigned long long* __restrict__ stats) {
  __shared__ int cand[UDH_EXPOSURE_MAX_FRAMES];
  __shared__ int wcount[8], nchunks;
  __shared__ uchar4 val[2 * EX_CHUNK][256];                             // .w: valid
  __shared__ short2 blk[2 * EX_CHUNK][256];
  __shared__ long long soff[EX_PAIRS];                                  // the slot's cell offset, -1: no listed pair
  __shared__ int snx[EX_PAIRS], sb0[EX_PAIRS][4];                       // cells per row; bx_i0, by_i0, bx_j0, by_j0
  const int tx0 = blockIdx.x * EX_TILE_W, ty0 = blockIdx.y * EX_TILE_H;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nc = ex_candidates(fr, n, tx0, ty0, cand, wcount);
  // the chunk count is re-read from shared memory: kept in a register it lives across the warp's double-division call
  // and ptxas spills it
  if (threadIdx.x == 0) nchunks = (nc + EX_CHUNK - 1) / EX_CHUNK;
  __syncthreads();
  for (int A = 0; A < *(volatile int*)&nchunks; ++A) {
    for (int B = A; B < *(volatile int*)&nchunks; ++B) {
      if (threadIdx.x < EX_PAIRS) {
        const int a = threadIdx.x / EX_CHUNK, b = threadIdx.x % EX_CHUNK, ka = A * EX_CHUNK + a, kb = B * EX_CHUNK + b;
        long long o = -1;
        if (ka < nc && kb < nc && (A != B || a <= b)) {
          const int i = cand[ka], j = cand[kb], lo = ex_pair(pair_ptr, pair_j, i, j);
          if (lo >= 0) {
            const ExposureBlockFrame *Fi = fr + i, *Fj = fr + j;
            const int x0 = max(__ldg(&Fi->rx), __ldg(&Fj->rx)), y0 = max(__ldg(&Fi->ry), __ldg(&Fj->ry));
            o = __ldg(cell_off + lo);
            snx[threadIdx.x] = __ldg(cell_nx + lo);
            sb0[threadIdx.x][0] = (x0 - __ldg(&Fi->rx)) / __ldg(&Fi->bkw);
            sb0[threadIdx.x][1] = (y0 - __ldg(&Fi->ry)) / __ldg(&Fi->bkh);
            sb0[threadIdx.x][2] = (x0 - __ldg(&Fj->rx)) / __ldg(&Fj->bkw);
            sb0[threadIdx.x][3] = (y0 - __ldg(&Fj->ry)) / __ldg(&Fj->bkh);
          }
        }
        soff[threadIdx.x] = o;
      }
      __syncthreads();
      const int nA = min(EX_CHUNK, nc - A * EX_CHUNK), nB = A == B ? 0 : min(EX_CHUNK, nc - B * EX_CHUNK);
      for (int r = warp; r < EX_TILE_H; r += 8) {
        const int x = tx0 + lane, y = ty0 + r;
        for (int q = 0; q < nA + nB; ++q) {
          const int k = cand[q < nA ? A * EX_CHUNK + q : B * EX_CHUNK + q - nA];
          const ExposureBlockFrame* F = fr + k;
          const int sx = x - __ldg(&F->rx), sy = y - __ldg(&F->ry);
          int v[3] = {0, 0, 0};
          bool ok = false;
          int bx = 0, by = 0;
          if ((unsigned)sx < (unsigned)__ldg(&F->rw) && (unsigned)sy < (unsigned)__ldg(&F->rh)) {
            double mi[9];
#pragma unroll
            for (int t = 0; t < 9; ++t) mi[t] = __ldg(F->mi + t);
            const uint8_t* s = reinterpret_cast<const uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&F->src)));
            ok = mb_roi_warp(s, __ldg(&F->h), __ldg(&F->w), mi, sx, sy, __ldg(&F->bw), v);
            bx = sx / __ldg(&F->bkw);
            by = sy / __ldg(&F->bkh);
            const int64_t b = __ldg(&F->boff) + (int64_t)by * __ldg(&F->bpx) + bx;
            for (int f = 0; f < feeds; ++f) {
#pragma unroll
              for (int c = 0; c < 3; ++c) v[c] = ex_apply(v[c], __ldg(hist + ((int64_t)f * nblocks + b) * 3 + c));
            }
          }
          const int slot = q < nA ? q : EX_CHUNK + q - nA;
          val[slot][threadIdx.x] = make_uchar4(v[0], v[1], v[2], ok);
          blk[slot][threadIdx.x] = make_short2((short)bx, (short)by);
        }
        __syncwarp();
        for (int t = 0; t < EX_PAIRS; ++t) {
          const long long o = soff[t];
          if (o < 0) continue;
          const int a = t / EX_CHUNK, b = A == B ? t % EX_CHUNK : EX_CHUNK + t % EX_CHUNK;
          const uchar4 u = val[a][threadIdx.x], w = val[b][threadIdx.x];
          const bool both = u.w && w.w;
          if (!__any_sync(0xffffffffu, both)) continue;
          const short2 bu = blk[a][threadIdx.x], bv = blk[b][threadIdx.x];
          const int cell = (int)o + (bu.y - sb0[t][1] + bv.y - sb0[t][3]) * snx[t] + (bu.x - sb0[t][0] + bv.x - sb0[t][2]);
          const unsigned grp = __match_any_sync(0xffffffffu, both ? cell : -1);
          const bool leader = both && lane == __ffs(grp) - 1;         // lanes without the pair form one group that adds nothing
          unsigned long long* dst = stats + (int64_t)cell * UDH_EXPOSURE_STATS;
          auto add = [&](int q, unsigned v) {
            const unsigned tot = __reduce_add_sync(grp, v);                // < 2^26: 32 lanes of < 2^21
            if (leader && tot) atomicAdd(dst + q, (unsigned long long)tot);
          };
          add(0, 1u);
          add(1, u.x); add(2, u.y); add(3, u.z);
          add(4, w.x); add(5, w.y); add(6, w.z);
          if (norms) {
            const uint64_t qu = __double2ull_rn(__dmul_rn(__dsqrt_rn((double)(u.x * u.x + u.y * u.y + u.z * u.z)), 0x1p52));
#pragma unroll
            for (int l = 0; l < 3; ++l) add(7 + l, (unsigned)(qu >> (21 * l)) & 0x1fffffu);
            const uint64_t qw = __double2ull_rn(__dmul_rn(__dsqrt_rn((double)(w.x * w.x + w.y * w.y + w.z * w.z)), 0x1p52));
#pragma unroll
            for (int l = 0; l < 3; ++l) add(10 + l, (unsigned)(qw >> (21 * l)) & 0x1fffffu);
          }
        }
        __syncwarp();
      }
      __syncthreads();
    }
  }
}

// Jacobi-preconditioned conjugate gradients in one CTA.  Each thread owns rows tid, tid + blockDim.x, ..; every reduction
// is a fixed butterfly per warp and then over the warps, so all threads see the same bits and the run repeats exactly.
constexpr int SOLVE_THREADS = 1024;

__device__ __forceinline__ double2 solve_sum2(double2 v, double2* red) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    v.x += __shfl_xor_sync(0xffffffffu, v.x, o);
    v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < (int)(blockDim.x >> 5) ? red[lane] : make_double2(0.0, 0.0);
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
      v.x += __shfl_xor_sync(0xffffffffu, v.x, o);
      v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
    }
    if (lane == 0) red[32] = v;
  }
  __syncthreads();
  v = red[32];
  __syncthreads();
  return v;
}

__device__ __forceinline__ double csr_row(const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ col,
                                          const double* __restrict__ val, const double* v, int i) {
  double s = 0.0;
  for (int e = __ldg(row_ptr + i); e < __ldg(row_ptr + i + 1); ++e) s += __ldg(val + e) * v[__ldg(col + e)];
  return s;
}

__global__ void __launch_bounds__(SOLVE_THREADS) gainblock_solve_kernel(int n, const int32_t* __restrict__ row_ptr,
                                                                             const int32_t* __restrict__ col,
                                                                             const double* __restrict__ val,
                                                                             const double* __restrict__ b, double tol, int max_iter,
                                                                             double* __restrict__ x, int64_t* __restrict__ info,
                                                                             double* __restrict__ r, double* __restrict__ p,
                                                                             double* __restrict__ q, double* __restrict__ dinv) {
  __shared__ double2 red[33];
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    x[i] = 1.0;
    double d = 0.0;
    for (int e = __ldg(row_ptr + i); e < __ldg(row_ptr + i + 1); ++e)
      if (__ldg(col + e) == i) d = __ldg(val + e);
    dinv[i] = 1.0 / d;
  }
  __syncthreads();
  double2 acc = make_double2(0.0, 0.0);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double ri = __ldg(b + i) - csr_row(row_ptr, col, val, x, i);
    r[i] = ri;
    p[i] = dinv[i] * ri;
    acc.x += ri * p[i];
    acc.y += __ldg(b + i) * __ldg(b + i);
  }
  const double2 s0 = solve_sum2(acc, red);
  double rz = s0.x;
  const double bn = sqrt(s0.y);
  acc = make_double2(0.0, 0.0);
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc.x += r[i] * r[i];
  double rel = sqrt(solve_sum2(acc, red).x) / bn;
  int it = 0;
  while (it < max_iter && rel > tol) {
    acc = make_double2(0.0, 0.0);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const double qi = csr_row(row_ptr, col, val, p, i);
      q[i] = qi;
      acc.x += p[i] * qi;
    }
    const double alpha = rz / solve_sum2(acc, red).x;
    acc = make_double2(0.0, 0.0);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      x[i] += alpha * p[i];
      const double ri = r[i] - alpha * q[i];
      r[i] = ri;
      acc.x += ri * ri;
      acc.y += ri * (dinv[i] * ri);
    }
    const double2 s = solve_sum2(acc, red);
    rel = sqrt(s.x) / bn;
    const double beta = s.y / rz;
    rz = s.y;
    for (int i = threadIdx.x; i < n; i += blockDim.x) p[i] = dinv[i] * r[i] + beta * p[i];
    __syncthreads();
    ++it;
  }
  if (threadIdx.x == 0) {
    info[0] = it;
    info[1] = __double_as_longlong(rel);
  }
}

// The gain maps: one CTA per frame, float32(gains) filtered twice in place (tmp holds each row pass).
__device__ __forceinline__ int gm_reflect(int i, int n) { return n == 1 ? 0 : i < 0 ? -i : i >= n ? 2 * n - 2 - i : i; }

__global__ void __launch_bounds__(256) gainblock_maps_kernel(const double* __restrict__ gains, const int4* __restrict__ fb, int ch,
                                                                 float* __restrict__ maps, float* __restrict__ tmp) {
  const int4 f = fb[blockIdx.x];                                      // bpx, bpy, boff (low, high)
  const int bpx = f.x, bpy = f.y;
  const int64_t boff = (int64_t)(unsigned)f.z | ((int64_t)f.w << 32);
  const int ne = bpx * bpy * ch;
  float* a = maps + boff * ch;
  float* t = tmp + boff * ch;
  for (int e = threadIdx.x; e < ne; e += blockDim.x) a[e] = (float)__ldg(gains + (boff + e / ch) * 3 + e % ch);
  __syncthreads();
  for (int pass = 0; pass < 2; ++pass) {
    for (int e = threadIdx.x; e < ne; e += blockDim.x) {
      const int c = e % ch, bx = e / ch % bpx, by = e / ch / bpx;
      const float* row = a + (int64_t)by * bpx * ch + c;
      t[e] = __fadd_rn(__fmul_rn(__fadd_rn(row[gm_reflect(bx - 1, bpx) * ch], row[gm_reflect(bx + 1, bpx) * ch]), 0.25f),
                       __fmul_rn(row[bx * ch], 0.5f));
    }
    __syncthreads();
    for (int e = threadIdx.x; e < ne; e += blockDim.x) {
      const int c = e % ch, bx = e / ch % bpx, by = e / ch / bpx;
      const float* cl = t + (int64_t)bx * ch + c;
      const int64_t st = (int64_t)bpx * ch;
      a[e] = __fadd_rn(__fmul_rn(__fadd_rn(cl[gm_reflect(by - 1, bpy) * st], cl[gm_reflect(by + 1, bpy) * st]), 0.25f),
                       __fmul_rn(cl[by * st], 0.5f));
    }
    __syncthreads();
  }
}

// ---- seam finding: cv2.detail's Voronoi seam finder on the ROI validity masks (the rule: oracle/seam.py) ---------------
// Every fed frame's mask lives on its ROI (rh x rw bytes at element offset off of a pool).  The pairs are visited on the host
// in cv2's order; each pair runs two kernels over its window (the ROIs' intersection grown by SEAM_GAP): the column pass
// gives each window pixel its distance along the column to the nearest unique pixel of either frame, and the row pass
// turns that into the exact L1 distance (min over x' of g(x') + |x - x'|, a prefix and a suffix minimum) and clears one
// frame's mask at every pixel of the intersection.  All in int32: SEAM_INF marks "no source" and survives the adds
// (distances are below 2^17, the window's sides below 32767 + 2 SEAM_GAP).
constexpr int SEAM_INF = 1 << 30, SEAM_SEGS = 16, SEAM_ROW_THREADS = 256;

// Every frame's ROI validity (udh_mosaic_multiband_u8's mask, mb_roi_warp's rule), 0 / 255, into both pools.
__global__ void __launch_bounds__(256) seam_valid_kernel(const SeamFrame* __restrict__ fr, const double* __restrict__ M,
                                                         uint8_t* __restrict__ seam, uint8_t* __restrict__ blend) {
  __shared__ double mi[9];
  const int k = blockIdx.y;
  if (threadIdx.x == 0) cv_invert3(M + (int64_t)k * 9, mi);
  __syncthreads();
  const SeamFrame* F = fr + k;
  const uint8_t* s = reinterpret_cast<const uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&F->src)));
  const int h = __ldg(&F->h), w = __ldg(&F->w), rw = __ldg(&F->rw), bw = __ldg(&F->bw), npx = rw * __ldg(&F->rh);
  const int64_t off = __ldg(&F->off);
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < npx; e += gridDim.x * blockDim.x) {
    const int y = e / rw, x = e - y * rw;
    int X, Y;
    const double Wd = wp_coords(mi, x, y, bw, X, Y);
    const uint8_t v = Wd != 0.0 && X >= 0 && X <= 32 * (w - 1) && Y >= 0 && Y <= 32 * (h - 1) ? 255 : 0;
    seam[off + e] = v;
    blend[off + e] = v;
  }
}

// The pair's unique pixels at window pixel (x, y): bit 0 frame a's, bit 1 frame b's (a pixel both masks hold is neither's).
__device__ __forceinline__ int seam_unique(const uint8_t* __restrict__ seam, const SeamRect& a, const SeamRect& b, int cx, int cy) {
  const bool sa = seam_at(seam, a, cx, cy), sb = seam_at(seam, b, cx, cy);
  return (sa && !sb ? 1 : 0) | (sb && !sa ? 2 : 0);
}

// Column pass: a CTA takes 32 window columns (one per lane, so every row's loads and stores are coalesced) and splits the
// window's height into SEAM_SEGS segments, one per warp.  Each thread first finds the first and last unique row of its
// segment for both frames; the CTA shares them, so every thread knows the nearest unique row above and below its segment;
// then it scans its segment down (distance to the nearest source above) and up (below) and stores the minimum, g.
__global__ void __launch_bounds__(32 * SEAM_SEGS) seam_column_kernel(const uint8_t* __restrict__ seam, SeamRect a, SeamRect b,
                                                                     int wx0, int wy0, int ww, int wh, int* __restrict__ ga,
                                                                     int* __restrict__ gb) {
  __shared__ int first[2][SEAM_SEGS][32], last[2][SEAM_SEGS][32];
  const int lane = threadIdx.x, seg = threadIdx.y, x = blockIdx.x * 32 + lane;
  const int len = (wh + SEAM_SEGS - 1) / SEAM_SEGS, y0 = min(seg * len, wh), y1 = min(y0 + len, wh);
  int fa = -1, la = -1, fb = -1, lb = -1;
  if (x < ww) {
    for (int y = y0; y < y1; ++y) {
      const int u = seam_unique(seam, a, b, wx0 + x, wy0 + y);
      if (u & 1) { if (fa < 0) fa = y; la = y; }
      if (u & 2) { if (fb < 0) fb = y; lb = y; }
    }
  }
  first[0][seg][lane] = fa; last[0][seg][lane] = la;
  first[1][seg][lane] = fb; last[1][seg][lane] = lb;
  __syncthreads();
  if (x >= ww) return;
  int up[2] = {-1, -1}, dn[2] = {-1, -1};                          // nearest unique row above / below the segment
#pragma unroll
  for (int f = 0; f < 2; ++f) {
    for (int q = 0; q < seg; ++q)
      if (last[f][q][lane] >= 0) up[f] = last[f][q][lane];
    for (int q = SEAM_SEGS - 1; q > seg; --q)
      if (first[f][q][lane] >= 0) dn[f] = first[f][q][lane];
  }
  int pa = up[0], pb = up[1];
  for (int y = y0; y < y1; ++y) {
    const int u = seam_unique(seam, a, b, wx0 + x, wy0 + y);
    if (u & 1) pa = y;
    if (u & 2) pb = y;
    const int64_t e = (int64_t)y * ww + x;
    ga[e] = pa >= 0 ? y - pa : SEAM_INF;
    gb[e] = pb >= 0 ? y - pb : SEAM_INF;
  }
  int na = dn[0], nb = dn[1];
  for (int y = y1 - 1; y >= y0; --y) {
    const int u = seam_unique(seam, a, b, wx0 + x, wy0 + y);
    if (u & 1) na = y;
    if (u & 2) nb = y;
    const int64_t e = (int64_t)y * ww + x;
    if (na >= 0) ga[e] = min(ga[e], na - y);
    if (nb >= 0) gb[e] = min(gb[e], nb - y);
  }
}

__device__ __forceinline__ int2 seam_min2(int2 p, int2 q) { return make_int2(min(p.x, q.x), min(p.y, q.y)); }

// The minimum of v over the CTA's threads before this one (INT_MAX for thread 0), and over all of them (tot).
__device__ __forceinline__ int2 seam_scan_exclusive(int2 v, int2* wtot, int2& tot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int2 u = make_int2(__shfl_up_sync(0xffffffffu, v.x, o), __shfl_up_sync(0xffffffffu, v.y, o));
    if (lane >= o) v = seam_min2(v, u);
  }
  int2 ex = make_int2(__shfl_up_sync(0xffffffffu, v.x, 1), __shfl_up_sync(0xffffffffu, v.y, 1));
  if (lane == 0) ex = make_int2(INT_MAX, INT_MAX);
  if (lane == 31) wtot[warp] = v;
  __syncthreads();
  tot = make_int2(INT_MAX, INT_MAX);
#pragma unroll
  for (int q = 0; q < SEAM_ROW_THREADS / 32; ++q) {
    if (q < warp) ex = seam_min2(ex, wtot[q]);
    tot = seam_min2(tot, wtot[q]);
  }
  __syncthreads();                                                  // wtot is rewritten by the next scan
  return ex;
}

// Row pass: one CTA per row of the intersection (window row SEAM_GAP + r).  d(x) = min(x + P(x), S(x) - x) with P the
// prefix minimum of g(x') - x' and S the suffix minimum of g(x') + x', both frames at once, 4 elements per thread per
// chunk; P goes to this row's scratch (pa, pb) on the forward sweep, S is formed on the backward sweep, which also clears,
// at every intersection pixel, frame b's mask where d_a < d_b and frame a's elsewhere (ties and two infinite distances).
__global__ void __launch_bounds__(SEAM_ROW_THREADS) seam_row_kernel(uint8_t* __restrict__ seam, SeamRect a, SeamRect b, int wx0,
                                                                    int wy0, int ww, int iw, const int* __restrict__ ga,
                                                                    const int* __restrict__ gb, int* __restrict__ pa,
                                                                    int* __restrict__ pb) {
  __shared__ int2 wtot[SEAM_ROW_THREADS / 32];
  const int y = SEAM_GAP + blockIdx.x;
  const int* ra = ga + (int64_t)y * ww;
  const int* rb = gb + (int64_t)y * ww;
  int* qa = pa + (int64_t)blockIdx.x * ww;
  int* qb = pb + (int64_t)blockIdx.x * ww;
  constexpr int CHUNK = 4 * SEAM_ROW_THREADS;
  int2 carry = make_int2(INT_MAX, INT_MAX), tot;
  for (int c0 = 0; c0 < ww; c0 += CHUNK) {
    int2 run[4], m = make_int2(INT_MAX, INT_MAX);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int x = c0 + 4 * threadIdx.x + q;
      if (x < ww) m = seam_min2(m, make_int2(ra[x] - x, rb[x] - x));
      run[q] = m;
    }
    const int2 ex = seam_min2(seam_scan_exclusive(m, wtot, tot), carry);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int x = c0 + 4 * threadIdx.x + q;
      if (x < ww) {
        const int2 p = seam_min2(run[q], ex);
        qa[x] = p.x;
        qb[x] = p.y;
      }
    }
    carry = seam_min2(carry, tot);
  }
  __syncthreads();                                                  // P of the whole row is in place
  carry = make_int2(INT_MAX, INT_MAX);
  for (int c0 = 0; c0 < ww; c0 += CHUNK) {                          // e = ww - 1 - x: the suffix is a prefix in e
    int2 run[4], m = make_int2(INT_MAX, INT_MAX);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int x = ww - 1 - (c0 + 4 * threadIdx.x + q);
      if (x >= 0) m = seam_min2(m, make_int2(ra[x] + x, rb[x] + x));
      run[q] = m;
    }
    const int2 ex = seam_min2(seam_scan_exclusive(m, wtot, tot), carry);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int x = ww - 1 - (c0 + 4 * threadIdx.x + q);
      if (x < SEAM_GAP || x >= SEAM_GAP + iw) continue;
      const int2 S = seam_min2(run[q], ex);
      int da = min(x + qa[x], S.x - x), db = min(x + qb[x], S.y - x);
      da = da >= SEAM_INF / 2 ? SEAM_INF : da;
      db = db >= SEAM_INF / 2 ? SEAM_INF : db;
      const int cx = wx0 + x, cy = wy0 + y;
      if (da < db)
        seam[b.off + (int64_t)(cy - b.ry) * b.rw + (cx - b.rx)] = 0;
      else
        seam[a.off + (int64_t)(cy - a.ry) * a.rw + (cx - a.rx)] = 0;
    }
    carry = seam_min2(carry, tot);
  }
}

// The blend masks, in place over the validity the pool holds: cv2.dilate(seam, 3 x 3 rectangle; pixels outside the ROI
// never win) AND the validity.
__global__ void __launch_bounds__(256) seam_blend_mask_kernel(const SeamFrame* __restrict__ fr, const uint8_t* __restrict__ seam,
                                                              uint8_t* __restrict__ blend) {
  const SeamFrame* F = fr + blockIdx.y;
  const int rw = __ldg(&F->rw), rh = __ldg(&F->rh), npx = rw * rh;
  const int64_t off = __ldg(&F->off);
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < npx; e += gridDim.x * blockDim.x) {
    if (!blend[off + e]) continue;
    const int y = e / rw, x = e - y * rw;
    bool on = false;
    for (int dy = -1; dy <= 1 && !on; ++dy)
      for (int dx = -1; dx <= 1; ++dx)
        if ((unsigned)(x + dx) < (unsigned)rw && (unsigned)(y + dy) < (unsigned)rh && seam[off + (int64_t)(y + dy) * rw + x + dx]) {
          on = true;
          break;
        }
    if (!on) blend[off + e] = 0;
  }
}

}  // namespace udh

using namespace udh;

extern "C" int udh_warp_perspective_u8(const uint8_t* src, const double* M, uint8_t* dst, int n, int h, int w, int c, int dst_h,
                                       int dst_w, void* stream) {
  UDH_REQUIRE(src && M && dst, "udh_warp_perspective_u8: null pointer");
  UDH_REQUIRE(c == 1 || c == 3, "udh_warp_perspective_u8: channels must be 1 or 3 (got %d)", c);
  // source positions are int16 in OpenCV's remap: sides below 32767 keep a saturated position outside the image
  UDH_REQUIRE(n >= 0 && n <= 65535 && h >= 1 && w >= 1 && h < 32767 && w < 32767 && dst_h >= 1 && dst_w >= 1 && dst_h < 32767 &&
                  dst_w < 32767,
              "udh_warp_perspective_u8: bad dimensions (n %d, %dx%d -> %dx%d)", n, h, w, dst_h, dst_w);
  if (n == 0) return UDH_OK;
  const int bw = warp_tile_w(dst_h, dst_w);
  const int groups = (dst_h * dst_w + 3) / 4;
  const dim3 grid((unsigned)((groups + 255) / 256), (unsigned)n);
  if (c == 3)
    warp_perspective_u8_kernel<3><<<grid, 256, 0, as_stream(stream)>>>(src, M, h, w, dst, dst_h, dst_w, bw);
  else
    warp_perspective_u8_kernel<1><<<grid, 256, 0, as_stream(stream)>>>(src, M, h, w, dst, dst_h, dst_w, bw);
  return check_launch("udh_warp_perspective_u8");
}

// The feathered blend's workspace: the frame table, then the mask table, then the map table.
extern "C" size_t udh_mosaic_workspace_bytes(int n) {
  return n > 0 ? mb_align((size_t)n * sizeof(MosaicFrame)) + mb_align((size_t)n * sizeof(SeamMask)) + (size_t)n * sizeof(GainMapDev) : 0;
}

// The table of n gain maps on the rectangles rois [n,4] (an empty rectangle: the frame has no map and counts nowhere).
static int gm_table(const udh_gain_map* maps, const int32_t* rois, int n, int dst_h, int dst_w, std::vector<GainMapDev>& out,
                    const char* what) {
  out.assign((size_t)n, GainMapDev{});
  for (int k = 0; k < n; ++k) {
    const int* r = rois + 4 * k;
    if (r[2] <= r[0] || r[3] <= r[1]) continue;
    UDH_REQUIRE(r[0] >= 0 && r[1] >= 0 && r[2] <= dst_w && r[3] <= dst_h, "%s: frame %d's rectangle (%d, %d)..(%d, %d) leaves the %dx%d canvas",
                what, k, r[0], r[1], r[2], r[3], dst_h, dst_w);
    const udh_gain_map& m = maps[k];
    UDH_REQUIRE(m.map && m.cols && m.rows && m.bpx >= 1 && m.bpy >= 1 && (m.channels == 1 || m.channels == 3),
                "%s: frame %d's gain map is malformed (%dx%d blocks, %d channels)", what, k, m.bpy, m.bpx, m.channels);
    out[(size_t)k] = GainMapDev{m, r[0], r[1], r[2] - r[0], r[3] - r[1]};
  }
  return UDH_OK;
}

using BlendKernel = void (*)(const MosaicFrame*, int, const int32_t*, const int32_t*, int, int, int, int, uint8_t*, uint8_t*, const double*,
                             const SeamMask*, const GainMapDev*);

// The feathered blend's instantiation for C channels and the optional inputs given (gains and maps exclude each other).
template <int C>
static BlendKernel blend_kernel(bool gain, bool masked, bool map) {
  if (map) return masked ? mosaic_blend_u8_kernel<C, false, true, true> : mosaic_blend_u8_kernel<C, false, false, true>;
  if (gain) return masked ? mosaic_blend_u8_kernel<C, true, true, false> : mosaic_blend_u8_kernel<C, true, false, false>;
  return masked ? mosaic_blend_u8_kernel<C, false, true, false> : mosaic_blend_u8_kernel<C, false, false, false>;
}

extern "C" int udh_mosaic_blend_u8(const uint8_t* const* frames, const int32_t* sizes, const double* M, const double* gains,
                                   const udh_gain_map* maps, const uint8_t* const* masks, const int32_t* rois, int n, int c,
                                   const int32_t* tile_ptr, const int32_t* tile_frames, int dst_h, int dst_w, int feather, uint8_t* dst,
                                   uint8_t* mask, void* ws, size_t ws_bytes, void* stream) {
  const char* what = "udh_mosaic_blend_u8";
  UDH_REQUIRE(tile_ptr && tile_frames && dst && mask && (n == 0 || (frames && sizes && M && ws)), "%s: null pointer", what);
  UDH_REQUIRE(c == 1 || c == 3, "%s: channels must be 1 or 3 (got %d)", what, c);
  UDH_REQUIRE(n >= 0 && n <= 65535 && dst_h >= 1 && dst_w >= 1 && dst_h < 32767 && dst_w < 32767,
              "%s: bad dimensions (n %d, canvas %dx%d)", what, n, dst_h, dst_w);
  UDH_REQUIRE(feather >= 0 && feather <= 1024, "%s: feather must be in [0, 1024] (got %d)", what, feather);
  UDH_REQUIRE(!(gains && maps), "%s: gains and maps exclude each other", what);
  UDH_REQUIRE(n == 0 || rois || !(masks || maps), "%s: masks and maps need rois", what);
  const size_t need = udh_mosaic_workspace_bytes(n);
  if (ws_bytes < need) {
    set_error("%s: workspace of %zu bytes, %zu needed", what, ws_bytes, need);
    return UDH_EWS;
  }
  std::vector<MosaicFrame> fr((size_t)n);
  for (int k = 0; k < n; ++k) {
    const int h = sizes[2 * k], w = sizes[2 * k + 1];
    UDH_REQUIRE(frames[k], "%s: frame %d is a null pointer", what, k);
    UDH_REQUIRE(h >= 1 && w >= 1 && h < 32767 && w < 32767, "%s: frame %d is %dx%d", what, k, h, w);
    fr[(size_t)k].src = frames[k];
    fr[(size_t)k].h = h;
    fr[(size_t)k].w = w;
  }
  std::vector<SeamMask> sm(masks ? (size_t)n : 0, SeamMask{nullptr, 0, 0, 0, 0});
  for (int k = 0; k < (int)sm.size(); ++k) {
    const int* r = rois + 4 * k;
    if (r[2] <= r[0] || r[3] <= r[1]) continue;
    UDH_REQUIRE(r[0] >= 0 && r[1] >= 0 && r[2] <= dst_w && r[3] <= dst_h,
                "%s: frame %d's mask rectangle (%d, %d)..(%d, %d) leaves the %dx%d canvas", what, k, r[0], r[1], r[2], r[3], dst_h, dst_w);
    UDH_REQUIRE(masks[k], "%s: frame %d's mask is a null pointer", what, k);
    sm[(size_t)k] = SeamMask{masks[k], r[0], r[1], r[2] - r[0], r[3] - r[1]};
  }
  std::vector<GainMapDev> gm;
  int rc = maps ? gm_table(maps, rois, n, dst_h, dst_w, gm, what) : UDH_OK;
  if (rc != UDH_OK) return rc;
  const cudaStream_t st = as_stream(stream);
  char* base = static_cast<char*>(ws);
  SeamMask* sm_d = reinterpret_cast<SeamMask*>(base + mb_align((size_t)n * sizeof(MosaicFrame)));
  GainMapDev* gm_d = reinterpret_cast<GainMapDev*>(reinterpret_cast<char*>(sm_d) + mb_align((size_t)n * sizeof(SeamMask)));
  if (n > 0) {
    if ((rc = upload(base, fr, st, what)) != UDH_OK || (masks && (rc = upload(sm_d, sm, st, what)) != UDH_OK) ||
        (maps && (rc = upload(gm_d, gm, st, what)) != UDH_OK))
      return rc;
    invert_kernel<<<(n + 127) / 128, 128, 0, st>>>(M, reinterpret_cast<MosaicFrame*>(base), n);
    if ((rc = check_launch("udh_mosaic_blend_u8 (inverses)")) != UDH_OK) return rc;
  }
  const dim3 grid((unsigned)((dst_w + UDH_MOSAIC_TILE_W - 1) / UDH_MOSAIC_TILE_W),
                  (unsigned)((dst_h + UDH_MOSAIC_TILE_H - 1) / UDH_MOSAIC_TILE_H));
  const BlendKernel kernel = c == 3 ? blend_kernel<3>(gains, masks, maps) : blend_kernel<1>(gains, masks, maps);
  kernel<<<grid, 256, 0, st>>>(reinterpret_cast<const MosaicFrame*>(base), n, tile_ptr, tile_frames, dst_h, dst_w, warp_tile_w(dst_h, dst_w),
                               32 * feather, dst, mask, gains, masks ? sm_d : nullptr, maps ? gm_d : nullptr);
  return check_launch(what);
}

// The multi-band blend's workspace: the plan's layout, then the map table (after the pyramid, whose offsets do not move).
extern "C" size_t udh_mosaic_multiband_workspace_bytes(const int32_t* rois, int n, int dst_h, int dst_w, int bands) {
  MultibandPlan p;
  return mb_plan(nullptr, rois, nullptr, n, dst_h, dst_w, bands, p) == UDH_OK ? p.total + (size_t)n * sizeof(GainMapDev) : 0;
}

extern "C" int udh_debug_multiband_layout(const int32_t* rois, int n, int dst_h, int dst_w, int bands, size_t off[MB_MAX_BANDS + 1],
                                          int dims[3]) {
  UDH_REQUIRE(off && dims, "udh_debug_multiband_layout: null pointer");
  MultibandPlan p;
  const int rc = mb_plan(nullptr, rois, nullptr, n, dst_h, dst_w, bands, p);
  if (rc != UDH_OK) return rc;
  for (int i = 0; i <= MB_MAX_BANDS; ++i) off[i] = i <= p.B ? p.off_acc[i] : 0;
  dims[0] = p.B;
  dims[1] = p.Hp;
  dims[2] = p.Wp;
  return UDH_OK;
}

extern "C" int udh_mosaic_multiband_u8(const uint8_t* const* frames, const int32_t* sizes, const double* M, const double* gains,
                                       const udh_gain_map* maps, const uint8_t* const* masks, const int32_t* rois, int n, int c, int dst_h,
                                       int dst_w, int bands, uint8_t* dst, uint8_t* mask, void* ws, size_t ws_bytes, void* stream) {
  const char* what = "udh_mosaic_multiband_u8";
  UDH_REQUIRE(frames && sizes && M && rois && dst && mask && ws, "%s: null pointer", what);
  UDH_REQUIRE(c == 3, "%s: channels must be 3 (got %d)", what, c);
  UDH_REQUIRE(!(gains && maps), "%s: gains and maps exclude each other", what);
  MultibandPlan p;
  int rc = mb_plan(frames, rois, sizes, n, dst_h, dst_w, bands, p);
  if (rc != UDH_OK) return rc;
  const size_t need = p.total + (size_t)n * sizeof(GainMapDev);
  if (ws_bytes < need) {
    set_error("%s: workspace of %zu bytes, %zu needed", what, ws_bytes, need);
    return UDH_EWS;
  }
  for (int k = 0; masks && k < n; ++k) {
    UDH_REQUIRE(masks[k], "%s: frame %d's mask is a null pointer", what, k);
    p.fr[(size_t)k].bmask = masks[k];
  }
  std::vector<GainMapDev> gm;
  if (maps && (rc = gm_table(maps, rois, n, dst_h, dst_w, gm, what)) != UDH_OK) return rc;
  const cudaStream_t st = as_stream(stream);
  char* base = static_cast<char*>(ws);
  GainMapDev* gm_d = reinterpret_cast<GainMapDev*>(base + p.total);
  if ((rc = upload(base, p.fr, st, what)) != UDH_OK || (maps && (rc = upload(gm_d, gm, st, what)) != UDH_OK)) return rc;
  const MultibandFrame* fr = reinterpret_cast<const MultibandFrame*>(base);
  uchar4* G = reinterpret_cast<uchar4*>(base + p.off_g);
  int16_t* Wt = reinterpret_cast<int16_t*>(base + p.off_w);
  auto acc = [&](int i) { return reinterpret_cast<short4*>(base + p.off_acc[i]); };
  auto R = [&](int i) { return reinterpret_cast<short4*>(base + p.off_r[i]); };
  {
    ProfScope ps(PROF_MB_BASE, st);
    (maps ? multiband_base_kernel<true> : multiband_base_kernel<false>)<<<dim3(mb_blocks(p.max_px[0]), (unsigned)n), 256, 0, st>>>(
        fr, M, gains, gm_d, G, Wt);
    if ((rc = check_launch("udh_mosaic_multiband_u8 (base)")) != UDH_OK) return rc;
  }
  {
    ProfScope ps(PROF_MB_DOWN, st);
    for (int i = 0; i < p.B; ++i) {
      multiband_down_kernel<<<dim3(mb_blocks(p.max_px[i + 1]), (unsigned)n), 256, 0, st>>>(fr, G, Wt, i);
      if ((rc = check_launch("udh_mosaic_multiband_u8 (pyrDown)")) != UDH_OK) return rc;
    }
  }
  {
    ProfScope ps(PROF_MB_ACC, st);
    for (int i = 0; i <= p.B; ++i) {
      const int cw = p.Wp >> i, ch = p.Hp >> i;
      const dim3 grid((unsigned)((cw + MB_TILE_W - 1) / MB_TILE_W), (unsigned)((ch + MB_TILE_H - 1) / MB_TILE_H));
      multiband_accumulate_kernel<<<grid, 256, 0, st>>>(fr, n, G, Wt, i, i == p.B, cw, ch, acc(i));
      if ((rc = check_launch("udh_mosaic_multiband_u8 (accumulate)")) != UDH_OK) return rc;
    }
  }
  ProfScope ps(PROF_MB_COLLAPSE, st);
  for (int i = p.B; i >= 1; --i) {
    const int cw = p.Wp >> i, ch = p.Hp >> i;
    multiband_collapse_kernel<false><<<mb_blocks((int64_t)cw * ch), 256, 0, st>>>(acc(i), i < p.B ? R(i + 1) : nullptr, cw, ch, R(i),
                                                                                 0, 0, nullptr, nullptr);
    if ((rc = check_launch("udh_mosaic_multiband_u8 (collapse)")) != UDH_OK) return rc;
  }
  multiband_collapse_kernel<true><<<mb_blocks((int64_t)dst_h * dst_w), 256, 0, st>>>(acc(0), p.B ? R(1) : nullptr, p.Wp, p.Hp, nullptr,
                                                                                     dst_h, dst_w, dst, mask);
  return check_launch("udh_mosaic_multiband_u8");
}

extern "C" size_t udh_mosaic_exposure_workspace_bytes(int n) { return n > 0 ? (size_t)n * sizeof(ExposureFrame) : 0; }

extern "C" int udh_mosaic_exposure_stats_u8(const uint8_t* const* frames, const int32_t* sizes, const double* M, const int32_t* rois,
                                            int n, const int32_t* pair_ptr, const int32_t* pair_j, int npairs, const double* history,
                                            int feeds, int norms, int dst_h, int dst_w, uint64_t* stats, void* ws, size_t ws_bytes,
                                            void* stream) {
  const char* what = "udh_mosaic_exposure_stats_u8";
  UDH_REQUIRE(frames && sizes && M && rois && pair_ptr && pair_j && stats && ws && (feeds == 0 || history), "%s: null pointer", what);
  UDH_REQUIRE(n >= 1 && n <= UDH_EXPOSURE_MAX_FRAMES && dst_h >= 1 && dst_w >= 1 && dst_h < 32767 && dst_w < 32767,
              "%s: bad dimensions (n %d of at most %d, canvas %dx%d)", what, n, UDH_EXPOSURE_MAX_FRAMES, dst_h, dst_w);
  UDH_REQUIRE(npairs >= n && npairs <= n * (n + 1) / 2 && feeds >= 0 && feeds <= UDH_EXPOSURE_MAX_FEEDS,
              "%s: %d pairs of %d frames, %d feeds (at most %d)", what, npairs, n, feeds, UDH_EXPOSURE_MAX_FEEDS);
  if (ws_bytes < udh_mosaic_exposure_workspace_bytes(n)) {
    set_error("%s: workspace of %zu bytes, %zu needed", what, ws_bytes, udh_mosaic_exposure_workspace_bytes(n));
    return UDH_EWS;
  }
  std::vector<ExposureFrame> host((size_t)n);
  int rc;
  for (int k = 0; k < n; ++k)
    if ((rc = roi_frame(frames, sizes, rois, k, dst_h, dst_w, host[(size_t)k], what)) != UDH_OK) return rc;
  const cudaStream_t st = as_stream(stream);
  if ((rc = upload(ws, host, st, what)) != UDH_OK) return rc;
  UDH_CUDA(cudaMemsetAsync(stats, 0, (size_t)npairs * UDH_EXPOSURE_STATS * sizeof(uint64_t), st));
  ExposureFrame* fr = static_cast<ExposureFrame*>(ws);
  invert_kernel<<<(n + 127) / 128, 128, 0, st>>>(M, fr, n);
  if ((rc = check_launch("udh_mosaic_exposure_stats_u8 (inverses)")) != UDH_OK) return rc;
  const dim3 grid((unsigned)((dst_w + EX_TILE_W - 1) / EX_TILE_W), (unsigned)((dst_h + EX_TILE_H - 1) / EX_TILE_H));
  exposure_stats_kernel<<<grid, 256, 0, st>>>(fr, n, pair_ptr, pair_j, history, feeds, norms,
                                              reinterpret_cast<unsigned long long*>(stats));
  return check_launch(what);
}

// The host's plan of one seam call: the frame table, the pairs in visiting order with their windows, and the workspace.
struct SeamPlan {
  std::vector<SeamFrame> fr;
  std::vector<int> pi, pj;
  int64_t max_px = 0, max_win = 0, max_inner = 0;
  size_t off_g, off_p, total;
};

static int seam_plan(const uint8_t* const* frames, const int32_t* rois, const int32_t* sizes, int n, const int32_t* pair_ptr,
                     const int32_t* pair_j, int dst_h, int dst_w, SeamPlan& p, const char* what) {
  UDH_REQUIRE(rois && pair_ptr && (pair_j || !pair_ptr[n]), "%s: null pointer", what);
  UDH_REQUIRE(n >= 1 && n <= UDH_SEAM_MAX_FRAMES && dst_h >= 1 && dst_w >= 1 && dst_h < 32767 && dst_w < 32767,
              "%s: bad dimensions (n %d of at most %d, canvas %dx%d)", what, n, UDH_SEAM_MAX_FRAMES, dst_h, dst_w);
  p.fr.assign((size_t)n, SeamFrame{});
  int64_t off = 0;
  for (int k = 0; k < n; ++k) {
    SeamFrame& F = p.fr[k];
    const int rc = roi_frame(frames, sizes, rois, k, dst_h, dst_w, F, what);
    if (rc != UDH_OK) return rc;
    F.off = off;
    off += (int64_t)F.rw * F.rh;
    if ((int64_t)F.rw * F.rh > p.max_px) p.max_px = (int64_t)F.rw * F.rh;
  }
  UDH_REQUIRE(pair_ptr[0] == 0, "%s: pair_ptr[0] is %d", what, pair_ptr[0]);
  for (int i = 0; i < n; ++i) {
    UDH_REQUIRE(pair_ptr[i + 1] >= pair_ptr[i], "%s: pair_ptr decreases at frame %d", what, i);
    for (int e = pair_ptr[i]; e < pair_ptr[i + 1]; ++e) {
      const int j = pair_j[e];
      UDH_REQUIRE(j > i && j < n && (e == pair_ptr[i] || j > pair_j[e - 1]),
                  "%s: pair (%d, %d) is out of order or range", what, i, j);
      const SeamFrame &A = p.fr[i], &B = p.fr[j];
      const int iw = std::min(A.rx + A.rw, B.rx + B.rw) - std::max(A.rx, B.rx), ih = std::min(A.ry + A.rh, B.ry + B.rh) - std::max(A.ry, B.ry);
      UDH_REQUIRE(iw > 0 && ih > 0, "%s: the ROIs of pair (%d, %d) do not intersect", what, i, j);
      const int64_t ww = iw + 2 * SEAM_GAP, wh = ih + 2 * SEAM_GAP;
      p.max_win = std::max(p.max_win, ww * wh);
      p.max_inner = std::max(p.max_inner, ww * ih);
      p.pi.push_back(i);
      p.pj.push_back(j);
    }
  }
  p.off_g = mb_align((size_t)n * sizeof(SeamFrame));
  p.off_p = mb_align(p.off_g + 2 * (size_t)p.max_win * sizeof(int));
  p.total = mb_align(p.off_p + 2 * (size_t)p.max_inner * sizeof(int));
  return UDH_OK;
}

extern "C" size_t udh_mosaic_seam_workspace_bytes(const int32_t* rois, int n, const int32_t* pair_ptr, const int32_t* pair_j,
                                                  int dst_h, int dst_w) {
  SeamPlan p;
  return seam_plan(nullptr, rois, nullptr, n, pair_ptr, pair_j, dst_h, dst_w, p, "udh_mosaic_seam_masks_u8") == UDH_OK ? p.total : 0;
}

extern "C" int udh_mosaic_seam_masks_u8(const uint8_t* const* frames, const int32_t* sizes, const double* M, const int32_t* rois, int n,
                                        const int32_t* pair_ptr, const int32_t* pair_j, int dst_h, int dst_w, uint8_t* seam,
                                        uint8_t* blend, void* ws, size_t ws_bytes, void* stream) {
  const char* what = "udh_mosaic_seam_masks_u8";
  UDH_REQUIRE(frames && sizes && M && seam && blend && ws, "%s: null pointer", what);
  SeamPlan p;
  int rc = seam_plan(frames, rois, sizes, n, pair_ptr, pair_j, dst_h, dst_w, p, what);
  if (rc != UDH_OK) return rc;
  if (ws_bytes < p.total) {
    set_error("%s: workspace of %zu bytes, %zu needed", what, ws_bytes, p.total);
    return UDH_EWS;
  }
  const cudaStream_t st = as_stream(stream);
  char* base = static_cast<char*>(ws);
  if ((rc = upload(base, p.fr, st, what)) != UDH_OK) return rc;
  const SeamFrame* fr = reinterpret_cast<const SeamFrame*>(base);
  int* ga = reinterpret_cast<int*>(base + p.off_g);
  int* gb = ga + p.max_win;
  int* pa = reinterpret_cast<int*>(base + p.off_p);
  int* pb = pa + p.max_inner;
  seam_valid_kernel<<<dim3(mb_blocks(p.max_px), (unsigned)n), 256, 0, st>>>(fr, M, seam, blend);
  if ((rc = check_launch("udh_mosaic_seam_masks_u8 (validity)")) != UDH_OK) return rc;
  for (size_t q = 0; q < p.pi.size(); ++q) {
    const SeamFrame &A = p.fr[p.pi[q]], &B = p.fr[p.pj[q]];
    const SeamRect a{A.off, A.rx, A.ry, A.rw, A.rh}, b{B.off, B.rx, B.ry, B.rw, B.rh};
    const int x0 = std::max(A.rx, B.rx), y0 = std::max(A.ry, B.ry);
    const int iw = std::min(A.rx + A.rw, B.rx + B.rw) - x0, ih = std::min(A.ry + A.rh, B.ry + B.rh) - y0;
    const int ww = iw + 2 * SEAM_GAP, wh = ih + 2 * SEAM_GAP, wx0 = x0 - SEAM_GAP, wy0 = y0 - SEAM_GAP;
    seam_column_kernel<<<(unsigned)((ww + 31) / 32), dim3(32, SEAM_SEGS), 0, st>>>(seam, a, b, wx0, wy0, ww, wh, ga, gb);
    if ((rc = check_launch("udh_mosaic_seam_masks_u8 (columns)")) != UDH_OK) return rc;
    seam_row_kernel<<<(unsigned)ih, SEAM_ROW_THREADS, 0, st>>>(seam, a, b, wx0, wy0, ww, iw, ga, gb, pa, pb);
    if ((rc = check_launch("udh_mosaic_seam_masks_u8 (rows)")) != UDH_OK) return rc;
  }
  seam_blend_mask_kernel<<<dim3(mb_blocks(p.max_px), (unsigned)n), 256, 0, st>>>(fr, seam, blend);
  return check_launch("udh_mosaic_seam_masks_u8 (blend masks)");
}

extern "C" size_t udh_mosaic_seam_gc_workspace_bytes(const int32_t* rois, int n, const int32_t* pair_ptr, const int32_t* pair_j,
                                                     int dst_h, int dst_w) {
  SeamPlan p;
  if (seam_plan(nullptr, rois, nullptr, n, pair_ptr, pair_j, dst_h, dst_w, p, "udh_mosaic_seam_gc_masks_u8") != UDH_OK) return 0;
  return gc_workspace_bytes(mb_align((size_t)n * sizeof(SeamFrame)), p.max_win, (int64_t)p.pi.size());
}

// The Voronoi call's plan, validity and blend masks around gc_seam_pairs (seam_gc.cu).
extern "C" int udh_mosaic_seam_gc_masks_u8(const uint8_t* const* frames, const int32_t* sizes, const double* M, const int32_t* rois,
                                           int n, const int32_t* pair_ptr, const int32_t* pair_j, int dst_h, int dst_w, uint8_t* seam,
                                           uint8_t* blend, int64_t* cut, void* ws, size_t ws_bytes, void* stream) {
  const char* what = "udh_mosaic_seam_gc_masks_u8";
  UDH_REQUIRE(frames && sizes && M && seam && blend && ws, "%s: null pointer", what);
  SeamPlan p;
  int rc = seam_plan(frames, rois, sizes, n, pair_ptr, pair_j, dst_h, dst_w, p, what);
  if (rc != UDH_OK) return rc;
  const size_t off = mb_align((size_t)n * sizeof(SeamFrame)), need = gc_workspace_bytes(off, p.max_win, (int64_t)p.pi.size());
  if (ws_bytes < need) {
    set_error("%s: workspace of %zu bytes, %zu needed", what, ws_bytes, need);
    return UDH_EWS;
  }
  const cudaStream_t st = as_stream(stream);
  char* base = static_cast<char*>(ws);
  if ((rc = upload(base, p.fr, st, what)) != UDH_OK) return rc;
  const SeamFrame* fr = reinterpret_cast<const SeamFrame*>(base);
  seam_valid_kernel<<<dim3(mb_blocks(p.max_px), (unsigned)n), 256, 0, st>>>(fr, M, seam, blend);
  if ((rc = check_launch("udh_mosaic_seam_gc_masks_u8 (validity)")) != UDH_OK) return rc;
  if ((rc = gc_seam_pairs(base, off, p.max_win, fr, p.fr, M, seam, p.pi, p.pj, cut, st, what)) != UDH_OK) return rc;
  seam_blend_mask_kernel<<<dim3(mb_blocks(p.max_px), (unsigned)n), 256, 0, st>>>(fr, seam, blend);
  return check_launch("udh_mosaic_seam_gc_masks_u8 (blend masks)");
}

extern "C" size_t udh_mosaic_exposure_block_workspace_bytes(int n) { return n > 0 ? (size_t)n * sizeof(ExposureBlockFrame) : 0; }

extern "C" int udh_mosaic_exposure_block_stats_u8(const uint8_t* const* frames, const int32_t* sizes, const double* M, const int32_t* rois,
                                                  int n, const int32_t* blocks, const int64_t* boff, int64_t nblocks,
                                                  const int32_t* pair_ptr, const int32_t* pair_j, int npairs, const int64_t* cell_off,
                                                  const int32_t* cell_nx, int64_t nslots, const double* history, int feeds, int norms,
                                                  int dst_h, int dst_w, uint64_t* stats, void* ws, size_t ws_bytes, void* stream) {
  const char* what = "udh_mosaic_exposure_block_stats_u8";
  UDH_REQUIRE(frames && sizes && M && rois && blocks && boff && pair_ptr && pair_j && cell_off && cell_nx && stats && ws &&
                  (feeds == 0 || history),
              "%s: null pointer", what);
  UDH_REQUIRE(n >= 1 && n <= UDH_EXPOSURE_MAX_FRAMES && dst_h >= 1 && dst_w >= 1 && dst_h < 32767 && dst_w < 32767,
              "%s: bad dimensions (n %d of at most %d, canvas %dx%d)", what, n, UDH_EXPOSURE_MAX_FRAMES, dst_h, dst_w);
  UDH_REQUIRE(npairs >= n && npairs <= n * (n + 1) / 2 && feeds >= 0 && feeds <= UDH_EXPOSURE_MAX_FEEDS,
              "%s: %d pairs of %d frames, %d feeds (at most %d)", what, npairs, n, feeds, UDH_EXPOSURE_MAX_FEEDS);
  UDH_REQUIRE(nblocks >= n && nblocks <= UDH_EXPOSURE_MAX_BLOCKS && nslots >= 1,
              "%s: %lld blocks (at most %d), %lld cells", what, (long long)nblocks, UDH_EXPOSURE_MAX_BLOCKS, (long long)nslots);
  if (ws_bytes < udh_mosaic_exposure_block_workspace_bytes(n)) {
    set_error("%s: workspace of %zu bytes, %zu needed", what, ws_bytes, udh_mosaic_exposure_block_workspace_bytes(n));
    return UDH_EWS;
  }
  std::vector<ExposureBlockFrame> host((size_t)n);
  int rc;
  for (int k = 0; k < n; ++k) {
    ExposureBlockFrame& F = host[(size_t)k];
    if ((rc = roi_frame(frames, sizes, rois, k, dst_h, dst_w, F, what)) != UDH_OK) return rc;
    F.bkw = blocks[4 * k];
    F.bkh = blocks[4 * k + 1];
    F.bpx = blocks[4 * k + 2];
    F.boff = boff[k];
    UDH_REQUIRE(F.bkw >= 1 && F.bkh >= 1 && F.bpx == (F.rw + F.bkw - 1) / F.bkw &&
                    blocks[4 * k + 3] == (F.rh + F.bkh - 1) / F.bkh && F.boff >= 0 && F.boff + (int64_t)F.bpx * blocks[4 * k + 3] <= nblocks,
                "%s: frame %d's blocks (%dx%d, %d per row, from %lld) do not tile its %dx%d ROI within %lld blocks", what, k, F.bkw,
                F.bkh, F.bpx, (long long)F.boff, F.rw, F.rh, (long long)nblocks);
  }
  const cudaStream_t st = as_stream(stream);
  if ((rc = upload(ws, host, st, what)) != UDH_OK) return rc;
  UDH_CUDA(cudaMemsetAsync(stats, 0, (size_t)nslots * UDH_EXPOSURE_STATS * sizeof(uint64_t), st));
  ExposureBlockFrame* fr = static_cast<ExposureBlockFrame*>(ws);
  invert_kernel<<<(n + 127) / 128, 128, 0, st>>>(M, fr, n);
  if ((rc = check_launch("udh_mosaic_exposure_block_stats_u8 (inverses)")) != UDH_OK) return rc;
  const dim3 grid((unsigned)((dst_w + EX_TILE_W - 1) / EX_TILE_W), (unsigned)((dst_h + EX_TILE_H - 1) / EX_TILE_H));
  gainblock_stats_kernel<<<grid, 256, 0, st>>>(fr, n, pair_ptr, pair_j, cell_off, cell_nx, history, nblocks, feeds, norms,
                                                    reinterpret_cast<unsigned long long*>(stats));
  return check_launch(what);
}

extern "C" size_t udh_exposure_block_solve_workspace_bytes(int n) { return n > 0 ? (size_t)4 * n * sizeof(double) : 0; }

extern "C" int udh_exposure_block_solve(int n, const int32_t* row_ptr, const int32_t* col, const double* val, const double* b,
                                        double tol, int max_iter, double* x, int64_t* info, void* ws, size_t ws_bytes, void* stream) {
  UDH_REQUIRE(row_ptr && col && val && b && x && info && ws, "udh_exposure_block_solve: null pointer");
  UDH_REQUIRE(n >= 1 && n <= UDH_EXPOSURE_MAX_BLOCKS && max_iter >= 0 && tol >= 0.0,
              "udh_exposure_block_solve: n %d (at most %d), max_iter %d, tol %g", n, UDH_EXPOSURE_MAX_BLOCKS, max_iter, tol);
  if (ws_bytes < udh_exposure_block_solve_workspace_bytes(n)) {
    set_error("udh_exposure_block_solve: workspace of %zu bytes, %zu needed", ws_bytes, udh_exposure_block_solve_workspace_bytes(n));
    return UDH_EWS;
  }
  double* w = static_cast<double*>(ws);
  gainblock_solve_kernel<<<1, SOLVE_THREADS, 0, as_stream(stream)>>>(n, row_ptr, col, val, b, tol, max_iter, x, info, w, w + n,
                                                                          w + 2 * (size_t)n, w + 3 * (size_t)n);
  return check_launch("udh_exposure_block_solve");
}

extern "C" size_t udh_exposure_gain_maps_workspace_bytes(int64_t nblocks, int channels) {
  return nblocks > 0 && (channels == 1 || channels == 3)
             ? mb_align((size_t)nblocks * channels * sizeof(float)) + (size_t)UDH_EXPOSURE_MAX_FRAMES * sizeof(int4)
             : 0;
}

extern "C" int udh_exposure_gain_maps(const double* gains, int n, const int32_t* blocks, const int64_t* boff, int64_t nblocks,
                                      int channels, float* maps, void* ws, size_t ws_bytes, void* stream) {
  UDH_REQUIRE(gains && blocks && boff && maps && ws, "udh_exposure_gain_maps: null pointer");
  UDH_REQUIRE(n >= 1 && n <= UDH_EXPOSURE_MAX_FRAMES && nblocks >= n && nblocks <= UDH_EXPOSURE_MAX_BLOCKS &&
                  (channels == 1 || channels == 3),
              "udh_exposure_gain_maps: %d frames, %lld blocks, %d channels", n, (long long)nblocks, channels);
  if (ws_bytes < udh_exposure_gain_maps_workspace_bytes(nblocks, channels)) {
    set_error("udh_exposure_gain_maps: workspace of %zu bytes, %zu needed", ws_bytes,
              udh_exposure_gain_maps_workspace_bytes(nblocks, channels));
    return UDH_EWS;
  }
  std::vector<int4> fb((size_t)n);
  for (int k = 0; k < n; ++k) {
    const int bpx = blocks[4 * k + 2], bpy = blocks[4 * k + 3];
    UDH_REQUIRE(bpx >= 1 && bpy >= 1 && boff[k] >= 0 && boff[k] + (int64_t)bpx * bpy <= nblocks,
                "udh_exposure_gain_maps: frame %d's %dx%d blocks from %lld exceed %lld", k, bpy, bpx, (long long)boff[k],
                (long long)nblocks);
    fb[(size_t)k] = make_int4(bpx, bpy, (int)(uint32_t)boff[k], (int)(boff[k] >> 32));
  }
  const cudaStream_t st = as_stream(stream);
  int4* fb_d = reinterpret_cast<int4*>(static_cast<char*>(ws) + mb_align((size_t)nblocks * channels * sizeof(float)));
  const int rc = upload(fb_d, fb, st, "udh_exposure_gain_maps");
  if (rc != UDH_OK) return rc;
  gainblock_maps_kernel<<<(unsigned)n, 256, 0, st>>>(gains, fb_d, channels, maps, static_cast<float*>(ws));
  return check_launch("udh_exposure_gain_maps");
}
