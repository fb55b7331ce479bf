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
#include <cstdint>

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

template <int C>
__device__ __forceinline__ void wp_pixel(const uint8_t* __restrict__ s, int h, int w, const double* mi, int x, int y, int bw,
                                         uint8_t* out) {
  const int xb = x - x % bw;
  const double dxb = (double)xb, dy = (double)y, dx1 = (double)(x - xb);
  const double X0 = __dadd_rn(__dadd_rn(__dmul_rn(mi[0], dxb), __dmul_rn(mi[1], dy)), mi[2]);
  const double Y0 = __dadd_rn(__dadd_rn(__dmul_rn(mi[3], dxb), __dmul_rn(mi[4], dy)), mi[5]);
  const double W0 = __dadd_rn(__dadd_rn(__dmul_rn(mi[6], dxb), __dmul_rn(mi[7], dy)), mi[8]);
  double W = __dadd_rn(W0, __dmul_rn(mi[6], dx1));
  W = W != 0.0 ? __ddiv_rn(32.0, W) : 0.0;
  const int X = wp_fixed(__dadd_rn(X0, __dmul_rn(mi[0], dx1)), W);
  const int Y = wp_fixed(__dadd_rn(Y0, __dmul_rn(mi[3], dx1)), W);
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
  for (int c = 0; c < C; ++c) out[c] = (uint8_t)((acc[c] + (1 << 14)) >> 15);
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
