// Direct-method baseline: OpenCV's findTransformECC with MOTION_HOMOGRAPHY (code/utils/direct_homography.py:8-57) as the
// reference's conventional harness calls it (code/homography_conventional_synthetic.py:186-223), batched on the device.
//   ecc_prep_kernel     the uint8 gray planes the reference hands to cv2: augment (fp32) -> normalise with I's statistics
//                       (fp32) -> denorm_img (fp64) -> astype(uint8) (truncation) -> cvtColor(RGB2GRAY) (fixed point)
//   ecc_blur_kernel     pre-pass: OpenCV's 5x5 Gaussian (sigma 0 -> [1,4,6,4,1]/16), BORDER_REFLECT_101, into fp32.  On
//                       8-bit inputs every partial sum is a multiple of 1/256 below 256, so the blur is exact in fp32
//   ecc_iterate_kernel  one CTA per sample runs every iteration in one launch; the image gradients are recomputed from
//                       the blurred plane during the warp (DESIGN §5 row E)
//   ecc_h4p_kernel      pred_h4p = perspectiveTransform(pts1, inv(W)) - pts1, the harness's clamp and failure rules
#include <cfloat>
#include <climits>

#include "common.cuh"

namespace udh {

__constant__ float kEccMean[3] = {118.93f, 113.97f, 102.60f};
__constant__ float kEccStd[3] = {69.85f, 68.81f, 72.45f};
__constant__ double kEccMean64[3] = {118.93, 113.97, 102.60};      // utils/utils.py:406-413 (float64 numpy arrays)
__constant__ double kEccStd64[3] = {69.85, 68.81, 72.45};

// ---- input preparation ------------------------------------------------------------------------------------------------
// Every step is a function of one uint8 value per (sample, image, channel), so it is tabulated once per CTA.
// gamma: pow in fp64 rounded once to fp32 (a correctly rounded powf, reproducible on the host); the rest is the fp32
// arithmetic of udh_prep_inputs_u8_ex.  denorm_img multiplies the fp32 value by a float64 std and adds a float64 mean in
// two roundings (no FMA), and astype(uint8) truncates.
__global__ void __launch_bounds__(256) ecc_prep_kernel(const uint8_t* __restrict__ I, const uint8_t* __restrict__ Ip,
                                                       const float* __restrict__ aug, uint8_t* __restrict__ gI,
                                                       uint8_t* __restrict__ gIp, int npx) {
  __shared__ uint8_t lut[2][3][256];
  const int b = blockIdx.y;
  const bool on = aug && aug[b * 11] != 0.0f;
  for (int i = threadIdx.x; i < 2 * 3 * 256; i += blockDim.x) {
    const int im = i / 768, c = (i / 256) % 3, x = i & 255;
    float v = (float)x;
    if (on) {
      const float* a = aug + b * 11 + 1 + im * 5;
      v = (float)pow((double)v, (double)a[0]);
      v = __fmul_rn(v, a[1]);
      v = __fmul_rn(v, a[2 + c]);
      v = fminf(fmaxf(v, 0.0f), 255.0f);
    }
    const float n = __fdiv_rn(__fsub_rn(v, kEccMean[c]), kEccStd[c]);
    const double d = __dadd_rn(__dmul_rn((double)n, kEccStd64[c]), kEccMean64[c]);
    const int t = (int)d;                                                  // truncation toward zero
    lut[im][c][x] = (uint8_t)(t < 0 ? 0 : (t > 255 ? 255 : t));
  }
  __syncthreads();
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < npx; o += gridDim.x * blockDim.x) {
    const uint8_t* p = I + ((size_t)b * npx + o) * 3;
    const uint8_t* q = Ip + ((size_t)b * npx + o) * 3;
    // cvtColor RGB2GRAY on 8-bit data: 15-bit fixed point, round half up
    gI[(size_t)b * npx + o] = (uint8_t)((lut[0][0][p[0]] * 9798 + lut[0][1][p[1]] * 19235 + lut[0][2][p[2]] * 3735 + 16384) >> 15);
    gIp[(size_t)b * npx + o] = (uint8_t)((lut[1][0][q[0]] * 9798 + lut[1][1][q[1]] * 19235 + lut[1][2][q[2]] * 3735 + 16384) >> 15);
  }
}

// ---- pre-pass ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int reflect101(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

// plane z = 0: template, z = 1: input image
__global__ void __launch_bounds__(256) ecc_blur_kernel(const uint8_t* __restrict__ tmpl, const uint8_t* __restrict__ input,
                                                       float* __restrict__ out, int H, int W) {
  const int b = blockIdx.y, z = blockIdx.z;
  const size_t npx = (size_t)H * W;
  const uint8_t* src = (z == 0 ? tmpl : input) + (size_t)b * npx;
  float* dst = out + ((size_t)z * gridDim.y + b) * npx;
  const float k[5] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f};
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < (int)npx; o += gridDim.x * blockDim.x) {
    const int y = o / W, x = o - y * W;
    int xs[5];
#pragma unroll
    for (int j = 0; j < 5; ++j) xs[j] = reflect101(x + j - 2, W);
    float acc = 0.0f;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const uint8_t* row = src + (size_t)reflect101(y + i - 2, H) * W;
      float r = 0.0f;
#pragma unroll
      for (int j = 0; j < 5; ++j) r += k[j] * (float)row[xs[j]];
      acc += k[i] * r;                                                     // exact: see the file header
    }
    dst[o] = acc;
  }
}

// ---- iterations -------------------------------------------------------------------------------------------------------
constexpr int kEccThreads = 512;
constexpr int kEccWarps = kEccThreads / 32;
constexpr int kEccAcc = 36 + 8 + 8 + 1;                                    // Hessian (upper), image / template projections, correlation

// 8x8 system with two right-hand sides, one warp: lane r < 8 owns row r = a[0..7] | a[8] a[9].  LU with partial pivoting
// (the first row of maximal |a[k]|) on shuffles, as the DLT kernel does; every lane returns both solutions.
__device__ __forceinline__ void lu_solve2_warp(double (&a)[10], double (&x0)[8], double (&x1)[8], int lane) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    double best = (lane >= k && lane < 8) ? fabs(a[k]) : -1.0;
    int idx = lane;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      const double ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
      if (ob > best || (ob == best && oi < idx)) { best = ob; idx = oi; }
    }
    const int piv = __shfl_sync(0xffffffffu, idx, 0);
    const int src = (lane == k) ? piv : ((lane == piv) ? k : lane);
#pragma unroll
    for (int c = k; c < 10; ++c) a[c] = __shfl_sync(0xffffffffu, a[c], src);
    double pk[10];
#pragma unroll
    for (int c = k; c < 10; ++c) pk[c] = __shfl_sync(0xffffffffu, a[c], k);
    if (lane > k && lane < 8) {
      const double f = a[k] / pk[k];
#pragma unroll
      for (int c = k + 1; c < 10; ++c) a[c] = fma(-f, pk[c], a[c]);
      a[k] = 0.0;
    }
  }
#pragma unroll
  for (int k = 7; k >= 0; --k) {
    const double u = __shfl_sync(0xffffffffu, a[8] / a[k], k);
    const double v = __shfl_sync(0xffffffffu, a[9] / a[k], k);
    x0[k] = u; x1[k] = v;
    if (lane < k) { a[8] = fma(-a[k], u, a[8]); a[9] = fma(-a[k], v, a[9]); }
  }
}

// Sum v[0..n) over the CTA in a fixed order (xor butterfly in each warp, then the warps in index order): the result does
// not depend on scheduling.  Every thread returns with tot[] valid.
template <int N>
__device__ __forceinline__ void cta_sum(double (&v)[N], double (*red)[kEccAcc], double* tot) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    double s = v[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[wid][k] = s;
  }
  __syncthreads();
  if (threadIdx.x < N) {
    double s = 0.0;
    for (int w = 0; w < kEccWarps; ++w) s += red[w][threadIdx.x];
    tot[threadIdx.x] = s;
  }
  __syncthreads();
}

struct EccWarp {          // where template pixel (x, y) lands in the input image under W (WARP_INVERSE_MAP: src = W (x, y, 1))
  int xi, yi;             // top-left source pixel of the bilinear footprint
  float ax, ay;           // its weights' fractions, multiples of 1/32 (warpPerspective's INTER_TAB_SIZE)
  bool mask;              // INTER_NEAREST sample of the all-ones pre-mask
};

__device__ __forceinline__ EccWarp ecc_map(const double (&M)[9], int x, int y, int H, int W) {
  const double X0 = M[0] * x + M[1] * y + M[2], Y0 = M[3] * x + M[4] * y + M[5], W0 = M[6] * x + M[7] * y + M[8];
  const double lo = (double)INT_MIN, hi = (double)INT_MAX;
  const double wl = W0 != 0.0 ? 32.0 / W0 : 0.0;
  const int X = __double2int_rn(fmax(lo, fmin(hi, X0 * wl))), Y = __double2int_rn(fmax(lo, fmin(hi, Y0 * wl)));
  const double wn = W0 != 0.0 ? 1.0 / W0 : 0.0;
  const int Xn = __double2int_rn(fmax(lo, fmin(hi, X0 * wn))), Yn = __double2int_rn(fmax(lo, fmin(hi, Y0 * wn)));
  EccWarp r;
  r.xi = max(-32768, min(32767, X >> 5));
  r.yi = max(-32768, min(32767, Y >> 5));
  r.ax = (float)(X & 31) * (1.0f / 32.0f);
  r.ay = (float)(Y & 31) * (1.0f / 32.0f);
  r.mask = Xn >= 0 && Xn < W && Yn >= 0 && Yn < H;
  return r;
}

__device__ __forceinline__ float ecc_px(const float* __restrict__ p, int x, int y, int H, int W) {
  return (x >= 0 && x < W && y >= 0 && y < H) ? __ldg(p + (size_t)y * W + x) : 0.0f;
}
// filter2D with [-0.5, 0, 0.5] (BORDER_REFLECT_101: zero on the first and last column / row), 0 outside the image
__device__ __forceinline__ float ecc_gx(const float* __restrict__ p, int x, int y, int H, int W) {
  if (x < 0 || x >= W || y < 0 || y >= H || x == 0 || x == W - 1) return 0.0f;
  return __fmul_rn(0.5f, __fsub_rn(__ldg(p + (size_t)y * W + x + 1), __ldg(p + (size_t)y * W + x - 1)));
}
__device__ __forceinline__ float ecc_gy(const float* __restrict__ p, int x, int y, int H, int W) {
  if (x < 0 || x >= W || y < 0 || y >= H || y == 0 || y == H - 1) return 0.0f;
  return __fmul_rn(0.5f, __fsub_rn(__ldg(p + (size_t)(y + 1) * W + x), __ldg(p + (size_t)(y - 1) * W + x)));
}
// remapBilinear's order: ((v00 w00 + v01 w01) + v10 w10) + v11 w11 with the exact table weights, no FMA
__device__ __forceinline__ float ecc_bilerp(float v00, float v01, float v10, float v11, float ax, float ay) {
  const float w00 = __fmul_rn(1.0f - ay, 1.0f - ax), w01 = __fmul_rn(1.0f - ay, ax);
  const float w10 = __fmul_rn(ay, 1.0f - ax), w11 = __fmul_rn(ay, ax);
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(v00, w00), __fmul_rn(v01, w01)), __fmul_rn(v10, w10)), __fmul_rn(v11, w11));
}

__global__ void __launch_bounds__(kEccThreads, 1) ecc_iterate_kernel(const float* __restrict__ blurred, const float* __restrict__ W_init,
                                                                     int max_iters, double eps, float* __restrict__ W_out,
                                                                     double* __restrict__ rho_out, int32_t* __restrict__ iters_out,
                                                                     int32_t* __restrict__ status_out, int B, int H, int W) {
  __shared__ double red[kEccWarps][kEccAcc];
  __shared__ double tot[kEccAcc];
  __shared__ float Wm[9];
  __shared__ double s_rho, s_last;
  __shared__ int s_status;
  const int b = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const size_t npx = (size_t)H * W;
  const float* T = blurred + (size_t)b * npx;                      // template (smoothed)
  const float* Im = blurred + ((size_t)B + b) * npx;               // input image (smoothed)
  if (threadIdx.x < 9) Wm[threadIdx.x] = W_init ? W_init[(size_t)b * 9 + threadIdx.x] : ((threadIdx.x & 3) == 0 ? 1.0f : 0.0f);
  if (threadIdx.x == 0) { s_rho = -1.0; s_last = -eps; s_status = 0; }
  __syncthreads();
  int it = 0;
  for (int i = 1; i <= max_iters && fabs(s_rho - s_last) >= eps; ++i) {
    it = i;
    double M[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) M[k] = (double)Wm[k];
    // pass 1: masked mean / standard deviation of the warped image and of the template (meanStdDev, fp64 sums)
    double st[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (int y = wid; y < H; y += kEccWarps)
      for (int x = lane; x < W; x += 32) {
        const EccWarp m = ecc_map(M, x, y, H, W);
        if (!m.mask) continue;
        const float iw = ecc_bilerp(ecc_px(Im, m.xi, m.yi, H, W), ecc_px(Im, m.xi + 1, m.yi, H, W), ecc_px(Im, m.xi, m.yi + 1, H, W),
                                    ecc_px(Im, m.xi + 1, m.yi + 1, H, W), m.ax, m.ay);
        const float t = __ldg(T + (size_t)y * W + x);
        st[0] += 1.0; st[1] += iw; st[2] += (double)iw * iw; st[3] += t; st[4] += (double)t * t;
      }
    cta_sum(st, red, tot);
    const double n = tot[0];
    const double mI = n > 0 ? tot[1] / n : 0.0, mT = n > 0 ? tot[3] / n : 0.0;
    const double sdI = n > 0 ? sqrt(fmax(tot[2] / n - mI * mI, 0.0)) : 0.0, sdT = n > 0 ? sqrt(fmax(tot[4] / n - mT * mT, 0.0)) : 0.0;
    const double imgNorm = sqrt(n * sdI * sdI), tmpNorm = sqrt(n * sdT * sdT);
    const float mIf = (float)mI, mTf = (float)mT;                    // subtract(Mat, Scalar) converts the mean to float
    // pass 2: Jacobian (image_jacobian_homo_ECC), Hessian, projections, correlation; fp32 partials per thread
    const float h0 = Wm[0], h1 = Wm[3], h2 = Wm[6], h3 = Wm[1], h4 = Wm[4], h5 = Wm[7], h6 = Wm[2], h7 = Wm[5];
    float acc[kEccAcc];
#pragma unroll
    for (int k = 0; k < kEccAcc; ++k) acc[k] = 0.0f;
    for (int y = wid; y < H; y += kEccWarps)
      for (int x = lane; x < W; x += 32) {
        const EccWarp m = ecc_map(M, x, y, H, W);
        const int x0 = m.xi, y0 = m.yi;
        if (x0 + 1 < 0 || x0 >= W || y0 + 1 < 0 || y0 >= H) continue;   // footprint outside: image, gradients, mask all 0
        const float iw = ecc_bilerp(ecc_px(Im, x0, y0, H, W), ecc_px(Im, x0 + 1, y0, H, W), ecc_px(Im, x0, y0 + 1, H, W),
                                    ecc_px(Im, x0 + 1, y0 + 1, H, W), m.ax, m.ay);
        const float gx = ecc_bilerp(ecc_gx(Im, x0, y0, H, W), ecc_gx(Im, x0 + 1, y0, H, W), ecc_gx(Im, x0, y0 + 1, H, W),
                                    ecc_gx(Im, x0 + 1, y0 + 1, H, W), m.ax, m.ay);
        const float gy = ecc_bilerp(ecc_gy(Im, x0, y0, H, W), ecc_gy(Im, x0 + 1, y0, H, W), ecc_gy(Im, x0, y0 + 1, H, W),
                                    ecc_gy(Im, x0 + 1, y0 + 1, H, W), m.ax, m.ay);
        const float iz = m.mask ? iw - mIf : iw;                         // outside the mask the warped image keeps its raw value
        const float tz = m.mask ? __ldg(T + (size_t)y * W + x) - mTf : 0.0f;
        const float xf = (float)x, yf = (float)y;
        const float den = xf * h2 + yf * h5 + 1.0f;
        const float hatX = (-xf * h0 - yf * h3 - h6) / den, hatY = (-xf * h1 - yf * h4 - h7) / den;
        const float gxd = gx / den, gyd = gy / den;
        const float tmp = hatX * gxd + hatY * gyd;
        const float J[8] = {gxd * xf, gyd * xf, tmp * xf, gxd * yf, gyd * yf, tmp * yf, gxd, gyd};
        int q = 0;
#pragma unroll
        for (int r = 0; r < 8; ++r)
#pragma unroll
          for (int c = r; c < 8; ++c) acc[q++] += J[r] * J[c];
#pragma unroll
        for (int r = 0; r < 8; ++r) { acc[36 + r] += J[r] * iz; acc[44 + r] += J[r] * tz; }
        acc[52] += tz * iz;
      }
    double accd[kEccAcc];
#pragma unroll
    for (int k = 0; k < kEccAcc; ++k) accd[k] = (double)acc[k];
    cta_sum(accd, red, tot);
    if (wid == 0) {
      const double corr = tot[52];
      const double rho = corr / (imgNorm * tmpNorm);
      double a[10], xi[8], xt[8];
      int q = 0, rowStart[8];
      for (int r = 0; r < 8; ++r) { rowStart[r] = q; q += 8 - r; }
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int r = lane < 8 ? lane : 0;
        const int lo = r < c ? r : c, hi = r < c ? c : r;
        a[c] = lane < 8 ? tot[rowStart[lo] + hi - lo] : 0.0;
      }
      a[8] = lane < 8 ? tot[36 + lane] : 0.0;
      a[9] = lane < 8 ? tot[44 + lane] : 0.0;
      lu_solve2_warp(a, xi, xt, lane);
      double ipH = 0.0, tpH = 0.0;
#pragma unroll
      for (int k = 0; k < 8; ++k) { ipH += tot[36 + k] * xi[k]; tpH += tot[44 + k] * xi[k]; }
      const double lambda_n = imgNorm * imgNorm - ipH, lambda_d = corr - tpH;
      int status = 0;
      if (isnan(rho)) status = UDH_ECC_NAN;
      else if (lambda_d <= 0.0) status = UDH_ECC_NOCONV;
      if (status == 0 && lane < 8) {
        const double lambda = lambda_n / lambda_d;
        const float dp = (float)(lambda * xt[lane] - xi[lane]);
        const int slot[8] = {0, 3, 6, 1, 4, 7, 2, 5};                     // update_warping_matrix_ECC's parameter order
        Wm[slot[lane]] += dp;
      }
      if (lane == 0) { s_last = s_rho; s_rho = rho; s_status = status; }
    }
    __syncthreads();
    if (s_status != 0) break;
  }
  if (threadIdx.x < 9) W_out[(size_t)b * 9 + threadIdx.x] = Wm[threadIdx.x];
  if (threadIdx.x == 0) {
    rho_out[b] = s_rho;
    iters_out[b] = it;
    status_out[b] = s_status;
  }
}

// ---- post-processing (direct_homography.py:42-57, homography_conventional_synthetic.py:204-223) -------------------------
__global__ void ecc_h4p_kernel(const float* __restrict__ Wm, const int32_t* __restrict__ status, const float* __restrict__ pts1,
                               const float* __restrict__ gt, float rho, float* __restrict__ pred, float* __restrict__ h_loss,
                               int32_t* __restrict__ fail, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float* w = Wm + (size_t)b * 9;
  const double m0 = w[0], m1 = w[1], m2 = w[2], m3 = w[3], m4 = w[4], m5 = w[5], m6 = w[6], m7 = w[7], m8 = w[8];
  const double c0 = m4 * m8 - m5 * m7, c1 = m5 * m6 - m3 * m8, c2 = m3 * m7 - m4 * m6;
  const double det = m0 * c0 + m1 * c1 + m2 * c2;
  const bool found = status[b] == 0 && det != 0.0 && isfinite(det);   // cv2 raised, or inv(W) failed: "not found"
  float p[8];
  if (found) {
    const double id = 1.0 / det;
    const double v[9] = {c0 * id, (m2 * m7 - m1 * m8) * id, (m1 * m5 - m2 * m4) * id,
                         c1 * id, (m0 * m8 - m2 * m6) * id, (m2 * m3 - m0 * m5) * id,
                         c2 * id, (m1 * m6 - m0 * m7) * id, (m0 * m4 - m1 * m3) * id};
#pragma unroll
    for (int k = 0; k < 4; ++k) {                                       // perspectiveTransform on float32 points
      const float x = pts1[b * 8 + 2 * k], y = pts1[b * 8 + 2 * k + 1];
      double s = x * v[6] + y * v[7] + v[8];
      float X = 0.0f, Y = 0.0f;
      if (fabs(s) > (double)FLT_EPSILON) {
        s = 1.0 / s;
        X = (float)((x * v[0] + y * v[1] + v[2]) * s);
        Y = (float)((x * v[3] + y * v[4] + v[5]) * s);
      }
      p[2 * k] = X - x; p[2 * k + 1] = Y - y;
    }
  } else {
#pragma unroll
    for (int k = 0; k < 8; ++k) p[k] = 0.0f;
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (p[k] >= rho) p[k] = 2.0f * rho;
    if (p[k] <= -rho) p[k] = -2.0f * rho;
    pred[(size_t)b * 8 + k] = p[k];
  }
  if (!gt) return;
  double se = 0.0, si = 0.0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const double g = gt[(size_t)b * 8 + k];
    se += ((double)p[k] - g) * ((double)p[k] - g);
    si += g * g;
  }
  double h = sqrt(se / 8.0);
  const double ident = sqrt(si / 8.0);
  int f = 0;
  if (!found) f = 1;
  else if (ident < h) { f = 2; h = ident; }
  if (h_loss) h_loss[b] = (float)h;
  if (fail) fail[b] = f;
}

}  // namespace udh

using namespace udh;

static size_t ecc_plane_floats(int B, int H, int W) { return (size_t)2 * B * H * W; }

extern "C" size_t udh_ecc_workspace_bytes(int B, int img_h, int img_w) {
  if (B < 1 || img_h < 2 || img_w < 2) return 0;
  return ecc_plane_floats(B, img_h, img_w) * sizeof(float);
}

extern "C" int udh_ecc_prep_u8(const uint8_t* I, const uint8_t* I_prime, const float* aug, uint8_t* gray_I, uint8_t* gray_I_prime, int B,
                               int img_h, int img_w, void* stream) {
  UDH_REQUIRE(I && I_prime && gray_I && gray_I_prime, "udh_ecc_prep_u8: null pointer");
  UDH_REQUIRE(B >= 1 && img_h >= 1 && img_w >= 1, "udh_ecc_prep_u8: bad dimensions");
  cudaStream_t st = as_stream(stream);
  ProfScope ps(PROF_ELTWISE, st);
  const int npx = img_h * img_w;
  dim3 grid(min((npx + 1023) / 1024, 256), B);
  ecc_prep_kernel<<<grid, 256, 0, st>>>(I, I_prime, aug, gray_I, gray_I_prime, npx);
  return check_launch("udh_ecc_prep_u8");
}

extern "C" int udh_ecc_homography(const uint8_t* tmpl, const uint8_t* input, const float* W_init, int max_iters, double eps, float* W,
                                  double* rho, int32_t* iters, int32_t* status, void* ws, size_t ws_bytes, int B, int img_h, int img_w,
                                  void* stream) {
  UDH_REQUIRE(tmpl && input && W && rho && iters && status && ws, "udh_ecc_homography: null pointer");
  UDH_REQUIRE(B >= 1 && img_h >= 2 && img_w >= 2 && img_h < 32768 && img_w < 32768, "udh_ecc_homography: bad dimensions");
  UDH_REQUIRE(max_iters >= 0, "udh_ecc_homography: negative iteration count");
  if (ws_bytes < udh_ecc_workspace_bytes(B, img_h, img_w)) {
    set_error("udh_ecc_homography: workspace of %zu bytes, %zu needed", ws_bytes, udh_ecc_workspace_bytes(B, img_h, img_w));
    return UDH_EWS;
  }
  cudaStream_t st = as_stream(stream);
  float* blurred = static_cast<float*>(ws);
  const int npx = img_h * img_w;
  ecc_blur_kernel<<<dim3(min((npx + 255) / 256, 128), B, 2), 256, 0, st>>>(tmpl, input, blurred, img_h, img_w);
  int rc = check_launch("ecc_blur");
  if (rc) return rc;
  ecc_iterate_kernel<<<B, kEccThreads, 0, st>>>(blurred, W_init, max_iters, eps, W, rho, iters, status, B, img_h, img_w);
  return check_launch("udh_ecc_homography");
}

extern "C" int udh_ecc_h4p(const float* W, const int32_t* status, const float* pts1, const float* gt, float rho_clamp, float* pred_h4p,
                           float* h_loss, int32_t* fail, int B, void* stream) {
  UDH_REQUIRE(W && status && pts1 && pred_h4p, "udh_ecc_h4p: null pointer");
  UDH_REQUIRE(gt || (!h_loss && !fail), "udh_ecc_h4p: h_loss and fail need gt");
  UDH_REQUIRE(B >= 0, "udh_ecc_h4p: negative batch");
  if (B == 0) return UDH_OK;
  ecc_h4p_kernel<<<(B + 127) / 128, 128, 0, as_stream(stream)>>>(W, status, pts1, gt, rho_clamp, pred_h4p, h_loss, fail, B);
  return check_launch("udh_ecc_h4p");
}
