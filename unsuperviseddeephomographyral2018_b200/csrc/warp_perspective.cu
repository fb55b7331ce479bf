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
// The sequence mosaic's blend (udh_mosaic_blend_u8, below) samples every frame with the same coordinate and tap helpers.
#include <cstdint>
#include <vector>

#include "common.cuh"

namespace udh {

__device__ __forceinline__ void cv_invert3(const double* m, double* t) {
  auto dm = [](double a, double b) { return __dmul_rn(a, b); };
  auto cof = [&](int a, int b, int c, int d) { return __dsub_rn(dm(m[a], m[b]), dm(m[c], m[d])); };
  double det = __dadd_rn(__dsub_rn(dm(m[0], cof(4, 8, 5, 7)), dm(m[1], cof(3, 8, 5, 6))), dm(m[2], cof(3, 7, 4, 6)));
  if (det == 0.0) {
    for (int k = 0; k < 9; ++k) t[k] = 0.0;
    return;
  }
  const double d = __ddiv_rn(1.0, det);
  t[0] = dm(cof(4, 8, 5, 7), d); t[1] = dm(cof(2, 7, 1, 8), d); t[2] = dm(cof(1, 5, 2, 4), d);
  t[3] = dm(cof(5, 6, 3, 8), d); t[4] = dm(cof(0, 8, 2, 6), d); t[5] = dm(cof(2, 3, 0, 5), d);
  t[6] = dm(cof(3, 7, 4, 6), d); t[7] = dm(cof(1, 6, 0, 7), d); t[8] = dm(cof(0, 4, 1, 3), d);
}

__device__ __forceinline__ int wp_fixed(double num, double W) {
  const double f = fmax(-2147483648.0, fmin(2147483647.0, __dmul_rn(num, W)));
  return __double2int_rn(f);
}

// The source position of output pixel (x, y) in 1/32 pixel (X, Y); returns the denominator before 32 / W (0: cv2 lands on
// source pixel (0, 0)).
__device__ __forceinline__ double wp_coords(const double* mi, int x, int y, int bw, int& X, int& Y) {
  const int xb = x - x % bw;
  const double dxb = (double)xb, dy = (double)y, dx1 = (double)(x - xb);
  const double X0 = __dadd_rn(__dadd_rn(__dmul_rn(mi[0], dxb), __dmul_rn(mi[1], dy)), mi[2]);
  const double Y0 = __dadd_rn(__dadd_rn(__dmul_rn(mi[3], dxb), __dmul_rn(mi[4], dy)), mi[5]);
  const double W0 = __dadd_rn(__dadd_rn(__dmul_rn(mi[6], dxb), __dmul_rn(mi[7], dy)), mi[8]);
  const double Wd = __dadd_rn(W0, __dmul_rn(mi[6], dx1));
  const double W = Wd != 0.0 ? __ddiv_rn(32.0, Wd) : 0.0;
  X = wp_fixed(__dadd_rn(X0, __dmul_rn(mi[0], dx1)), W);
  Y = wp_fixed(__dadd_rn(Y0, __dmul_rn(mi[3], dx1)), W);
  return Wd;
}

// The bilinear value at (X, Y) (1/32 pixel) of an h x w source with C channels: 15-bit weights, taps outside read 0.
template <int C>
__device__ __forceinline__ void wp_sample(const uint8_t* __restrict__ s, int h, int w, int X, int Y, int* v) {
  const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767);
  const int fx = X & 31, fy = Y & 31;
  const int wt[4] = {(32 - fx) * (32 - fy) * 32, fx * (32 - fy) * 32, (32 - fx) * fy * 32, fx * fy * 32};
  int acc[C];
#pragma unroll
  for (int c = 0; c < C; ++c) acc[c] = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int tx = sx + (k & 1), ty = sy + (k >> 1);
    if ((unsigned)tx < (unsigned)w && (unsigned)ty < (unsigned)h) {
      const uint8_t* p = s + ((int64_t)ty * w + tx) * C;
#pragma unroll
      for (int c = 0; c < C; ++c) acc[c] += wt[k] * (int)__ldg(p + c);
    }
  }
#pragma unroll
  for (int c = 0; c < C; ++c) v[c] = (acc[c] + (1 << 14)) >> 15;
}

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
  double mi[9];                   // cv_invert3 of the frame's M (frame -> canvas), filled by mosaic_invert_kernel
  const uint8_t* src;
  int h, w;
};

__global__ void mosaic_invert_kernel(const double* __restrict__ M, MosaicFrame* fr, int n) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) cv_invert3(M + (int64_t)k * 9, fr[k].mi);
}

// Gather form: one CTA per UDH_MOSAIC_TILE_H x UDH_MOSAIC_TILE_W canvas tile, each thread four consecutive pixels of one
// row.  The thread walks the tile's candidate frames, adds wt * v and wt of every frame valid at its pixels into 64-bit
// registers and stores the pixels once: no atomics, no accumulation buffer.  Integer sums: the result does not depend on
// the frames' order.
template <int C>
__global__ void __launch_bounds__(256) mosaic_blend_u8_kernel(const MosaicFrame* __restrict__ fr, int n,
                                                              const int32_t* __restrict__ tile_ptr,
                                                              const int32_t* __restrict__ tile_frames, int dh, int dw, int bw,
                                                              int feather32, uint8_t* __restrict__ dst,
                                                              uint8_t* __restrict__ mask) {
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
      if (Wd != 0.0 && X >= 0 && X <= xm && Y >= 0 && Y <= ym) {
        const int wt = 1 + min(min(min(X, xm - X), min(Y, ym - Y)), feather32);
        int v[C];
        wp_sample<C>(s, h, w, X, Y, v);
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
  const int bh = dst_h < 16 ? dst_h : 16;
  const int bw = 1024 / bh < dst_w ? 1024 / bh : dst_w;
  const int groups = (dst_h * dst_w + 3) / 4;
  const dim3 grid((unsigned)((groups + 255) / 256), (unsigned)n);
  if (c == 3)
    warp_perspective_u8_kernel<3><<<grid, 256, 0, as_stream(stream)>>>(src, M, h, w, dst, dst_h, dst_w, bw);
  else
    warp_perspective_u8_kernel<1><<<grid, 256, 0, as_stream(stream)>>>(src, M, h, w, dst, dst_h, dst_w, bw);
  return check_launch("udh_warp_perspective_u8");
}

extern "C" size_t udh_mosaic_workspace_bytes(int n) { return n > 0 ? (size_t)n * sizeof(MosaicFrame) : 0; }

extern "C" int udh_mosaic_blend_u8(const uint8_t* const* frames, const int32_t* sizes, const double* M, int n, int c,
                                   const int32_t* tile_ptr, const int32_t* tile_frames, int dst_h, int dst_w, int feather,
                                   uint8_t* dst, uint8_t* mask, void* ws, size_t ws_bytes, void* stream) {
  UDH_REQUIRE(tile_ptr && tile_frames && dst && mask && (n == 0 || (frames && sizes && M && ws)), "udh_mosaic_blend_u8: null pointer");
  UDH_REQUIRE(c == 1 || c == 3, "udh_mosaic_blend_u8: channels must be 1 or 3 (got %d)", c);
  UDH_REQUIRE(n >= 0 && n <= 65535 && dst_h >= 1 && dst_w >= 1 && dst_h < 32767 && dst_w < 32767,
              "udh_mosaic_blend_u8: bad dimensions (n %d, canvas %dx%d)", n, dst_h, dst_w);
  UDH_REQUIRE(feather >= 0 && feather <= 1024, "udh_mosaic_blend_u8: feather must be in [0, 1024] (got %d)", feather);
  if (ws_bytes < udh_mosaic_workspace_bytes(n)) {
    set_error("udh_mosaic_blend_u8: workspace of %zu bytes, %zu needed", ws_bytes, udh_mosaic_workspace_bytes(n));
    return UDH_EWS;
  }
  const cudaStream_t st = as_stream(stream);
  if (n > 0) {
    std::vector<MosaicFrame> host((size_t)n);
    for (int k = 0; k < n; ++k) {
      const int h = sizes[2 * k], w = sizes[2 * k + 1];
      UDH_REQUIRE(frames[k], "udh_mosaic_blend_u8: frame %d is a null pointer", k);
      UDH_REQUIRE(h >= 1 && w >= 1 && h < 32767 && w < 32767, "udh_mosaic_blend_u8: frame %d is %dx%d", k, h, w);
      host[k].src = frames[k];
      host[k].h = h;
      host[k].w = w;
    }
    // pageable source: the copy is staged before this call returns, so `host` may go
      const cudaError_t e = cudaMemcpyAsync(ws, host.data(), (size_t)n * sizeof(MosaicFrame), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) {
      set_error("udh_mosaic_blend_u8: frame table copy: %s", cudaGetErrorString(e));
      return UDH_ECUDA;
    }
    mosaic_invert_kernel<<<(n + 127) / 128, 128, 0, st>>>(M, static_cast<MosaicFrame*>(ws), n);
    const int rc = check_launch("udh_mosaic_blend_u8 (inverses)");
    if (rc != UDH_OK) return rc;
  }
  const int bh = dst_h < 16 ? dst_h : 16;
  const int bw = 1024 / bh < dst_w ? 1024 / bh : dst_w;
  const dim3 grid((unsigned)((dst_w + UDH_MOSAIC_TILE_W - 1) / UDH_MOSAIC_TILE_W),
                  (unsigned)((dst_h + UDH_MOSAIC_TILE_H - 1) / UDH_MOSAIC_TILE_H));
  const MosaicFrame* fr = static_cast<const MosaicFrame*>(ws);
  if (c == 3)
    mosaic_blend_u8_kernel<3><<<grid, 256, 0, st>>>(fr, n, tile_ptr, tile_frames, dst_h, dst_w, bw, 32 * feather, dst, mask);
  else
    mosaic_blend_u8_kernel<1><<<grid, 256, 0, st>>>(fr, n, tile_ptr, tile_frames, dst_h, dst_w, bw, 32 * feather, dst, mask);
  return check_launch("udh_mosaic_blend_u8");
}
