// The dataset generator's per-pixel warp (gen_synthetic_data.py:63-64 -> numpy_spatial_transformer.py), in fp64, bit for bit:
//   gray      cv2.cvtColor(bgr, COLOR_RGB2GRAY) as the generator calls it on a BGR image: the 15-bit rule with the R weight on
//             channel 0 and the B weight on channel 2.
//   warp      x_t, y_t = np.linspace(-1, 1, n) (i * step + start, the last point exactly 1); np.dot(theta, grid) as NumPy's
//             float64 dot evaluates a 3x3 by 3xN product: fma(t2, 1, fma(t1, y, t0 * x)); x / t; (x + 1) * W / 2;
//             floor, clip, weights from the clipped corners; ((wa Ia + wb Ib) + wc Ic) + wd Id without FMA; astype(uint8):
//             truncation toward zero, wrapped modulo 256 (NaN and values outside int32 give 0).
// One thread per output pixel writes the gray plane, the warped BGR image and the warp of the gray plane (the gray of the
// four source pixels, not the gray of the warped colour).  oracle/gen_data.py restates it.
#include <algorithm>

#include "common.cuh"

namespace udh {

__device__ __forceinline__ int gen_gray(const uint8_t* p) { return (p[0] * 9798 + p[1] * 19235 + p[2] * 3735 + 16384) >> 15; }

__device__ __forceinline__ uint8_t gen_cast_u8(double v) {
  if (!(v > -2147483649.0 && v < 2147483648.0)) return 0;
  return (uint8_t)(__double2int_rz(v) & 255);
}

__device__ __forceinline__ double gen_linspace(int i, int n) {
  if (n > 1 && i == n - 1) return 1.0;
  const double step = n > 1 ? __ddiv_rn(2.0, (double)(n - 1)) : 0.0;
  return __dadd_rn(__dmul_rn((double)i, step), -1.0);
}

__global__ void __launch_bounds__(256) gen_warp_u8_kernel(const uint8_t* __restrict__ bgr, const double* __restrict__ theta, int h, int w,
                                                          uint8_t* __restrict__ gray, uint8_t* __restrict__ warped,
                                                          uint8_t* __restrict__ warped_gray) {
  const int n = blockIdx.y;
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= h * w) return;
  const int i = o / w, j = o - i * w;
  const uint8_t* src = bgr + (int64_t)n * h * w * 3;
  gray[(int64_t)n * h * w + o] = (uint8_t)gen_gray(src + (int64_t)o * 3);
  const double* t = theta + (int64_t)n * 9;
  const double xt = gen_linspace(j, w), yt = gen_linspace(i, h);
  const double X = __dadd_rn(__fma_rn(t[1], yt, __dmul_rn(t[0], xt)), t[2]);
  const double Y = __dadd_rn(__fma_rn(t[4], yt, __dmul_rn(t[3], xt)), t[5]);
  const double T = __dadd_rn(__fma_rn(t[7], yt, __dmul_rn(t[6], xt)), t[8]);
  const double x = __ddiv_rn(__dmul_rn(__dadd_rn(__ddiv_rn(X, T), 1.0), (double)w), 2.0);
  const double y = __ddiv_rn(__dmul_rn(__dadd_rn(__ddiv_rn(Y, T), 1.0), (double)h), 2.0);
  // np.floor(x).astype(int) + 1, clipped: in double first, so huge or NaN coordinates clip like NumPy's int64 values do
  const double fx = floor(x), fy = floor(y);
  const double x0 = fmin(fmax(fx, 0.0), (double)(w - 1)), x1 = fmin(fmax(fx + 1.0, 0.0), (double)(w - 1));
  const double y0 = fmin(fmax(fy, 0.0), (double)(h - 1)), y1 = fmin(fmax(fy + 1.0, 0.0), (double)(h - 1));
  const double wa = __dmul_rn(__dsub_rn(x1, x), __dsub_rn(y1, y));
  const double wb = __dmul_rn(__dsub_rn(x1, x), __dsub_rn(y, y0));
  const double wc = __dmul_rn(__dsub_rn(x, x0), __dsub_rn(y1, y));
  const double wd = __dmul_rn(__dsub_rn(x, x0), __dsub_rn(y, y0));
  const int ix0 = (int)x0, ix1 = (int)x1, iy0 = (int)y0, iy1 = (int)y1;
  const uint8_t* pa = src + ((int64_t)iy0 * w + ix0) * 3;
  const uint8_t* pb = src + ((int64_t)iy1 * w + ix0) * 3;
  const uint8_t* pc = src + ((int64_t)iy0 * w + ix1) * 3;
  const uint8_t* pd = src + ((int64_t)iy1 * w + ix1) * 3;
  auto blend = [&](int a, int b, int c, int d) {
    return gen_cast_u8(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(wa, (double)a), __dmul_rn(wb, (double)b)), __dmul_rn(wc, (double)c)),
                                 __dmul_rn(wd, (double)d)));
  };
  uint8_t* dst = warped + ((int64_t)n * h * w + o) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) dst[c] = blend(pa[c], pb[c], pc[c], pd[c]);
  warped_gray[(int64_t)n * h * w + o] = blend(gen_gray(pa), gen_gray(pb), gen_gray(pc), gen_gray(pd));
}

__global__ void __launch_bounds__(256) gray_u8_kernel(const uint8_t* __restrict__ bgr, int64_t npx, uint8_t* __restrict__ gray) {
  for (int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; o < npx; o += (int64_t)gridDim.x * blockDim.x)
    gray[o] = (uint8_t)gen_gray(bgr + o * 3);
}

}  // namespace udh

using namespace udh;

extern "C" int udh_gen_warp_u8(const uint8_t* bgr, const double* theta, int n, int h, int w, uint8_t* gray, uint8_t* warped,
                               uint8_t* warped_gray, void* stream) {
  UDH_REQUIRE(bgr && theta && gray && warped && warped_gray, "udh_gen_warp_u8: null pointer");
  UDH_REQUIRE(n >= 0 && n <= 65535 && h >= 1 && w >= 1 && (int64_t)h * w < INT32_MAX, "udh_gen_warp_u8: bad dimensions");
  if (n == 0) return UDH_OK;
  gen_warp_u8_kernel<<<dim3((h * w + 255) / 256, n), 256, 0, as_stream(stream)>>>(bgr, theta, h, w, gray, warped, warped_gray);
  return check_launch("udh_gen_warp_u8");
}

extern "C" int udh_gray_u8(const uint8_t* bgr, int64_t npx, uint8_t* gray, void* stream) {
  UDH_REQUIRE(bgr && gray && npx >= 0, "udh_gray_u8: bad argument");
  if (npx == 0) return UDH_OK;
  gray_u8_kernel<<<(int)std::min<int64_t>((npx + 255) / 256, 8192), 256, 0, as_stream(stream)>>>(bgr, npx, gray);
  return check_launch("udh_gray_u8");
}
