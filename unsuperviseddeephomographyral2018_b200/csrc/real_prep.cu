// Real-data input pipeline (code/dataloader.py:146-200) and the real-data direct-method metric
// (code/homography_conventional_real.py:213-246), bit-identical to the host arithmetic they replace.
//   resize_up_u8_kernel      cv2.resize(uint8, INTER_AREA) to a larger size: linear interpolation with area coefficients,
//                            11-bit fixed point, VResizeLinearVec_32s8u's rounding.  Integer arithmetic: exact.  With
//                            INTER_LINEAR's table (udh_resize_linear_u8) it is cv2.resize(uint8, INTER_LINEAR), up or down.
//   real_prep_kernel         full-size uint8 I, I' -> the four network-size fp32 images of the loader (plain and augmented,
//                            normalised, INTER_AREA-downscaled).  Augment + normalise is a per-value table built on the host;
//                            the downscale is OpenCV's generic resizeArea in its summation order, each step rounded (no FMA).
//   ecc_corr_h4p_kernel      perspectiveTransform(corr1, W) - corr1, clamp to +-80, RMSE against corr2, failure rules.
#include <cfloat>

#include "common.cuh"

namespace udh {

// ---- uint8 upscale -------------------------------------------------------------------------------------------------------
// tab (int32): xsrc[dw], xa0[dw], xa1[dw], ysrc[dh], ya0[dh], ya1[dh]; one thread per output pixel (3 channels).
// ROW_PAIR: a further ysrc1[dh] gives the second source row.  INTER_LINEAR keeps the vertical coefficients at the borders
// and clamps both rows (rows -1 and 0 at the top are row 0 twice), which "the row after ysrc" cannot express.
template <bool ROW_PAIR>
__global__ void __launch_bounds__(256) resize_up_u8_kernel(const uint8_t* __restrict__ src, const int32_t* __restrict__ tab,
                                                           uint8_t* __restrict__ dst, int sh, int sw, int dh, int dw) {
  const int n = blockIdx.y;
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= dh * dw) return;
  const int dy = o / dw, dx = o - dy * dw;
  const int32_t *xs = tab, *xa0 = tab + dw, *xa1 = tab + 2 * dw;
  const int32_t *ys = tab + 3 * dw, *ya0 = ys + dh, *ya1 = ys + 2 * dh;
  const int sx = xs[dx], nx = min(sx + 1, sw - 1), sy = ys[dy], ny = ROW_PAIR ? ys[3 * dh + dy] : min(sy + 1, sh - 1);
  const int a0 = xa0[dx], a1 = xa1[dx], b0 = ya0[dy], b1 = ya1[dy];
  const uint8_t* r0 = src + ((size_t)n * sh + sy) * sw * 3;
  const uint8_t* r1 = src + ((size_t)n * sh + ny) * sw * 3;
  uint8_t* d = dst + (((size_t)n * dh + dy) * dw + dx) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int h0 = r0[sx * 3 + c] * a0 + r0[nx * 3 + c] * a1;       // horizontal pass of source rows sy and sy + 1
    const int h1 = r1[sx * 3 + c] * a0 + r1[nx * 3 + c] * a1;
    const int v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
    d[c] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
  }
}

// ---- full size uint8 -> network size fp32 --------------------------------------------------------------------------------
// luts [B][4][256][3]: plain I, plain I', augmented I, augmented I' (output t reads image t & 1 through table t).
// tab (int32, nullable = same size): nx, ny, then xofs[W+1], xsrc[nx], xw[nx] (fp32 bits), yofs[Hh+1], ysrc[ny], yw[ny]
// (fp32 bits): the entries of output column dx are [xofs[dx], xofs[dx+1]), in OpenCV's table order.
// One CTA per band of output rows of one sample.  STAGED: the source rows of the current output row are staged in shared
// memory; otherwise (they do not fit: camera frames, e.g. 14 rows of 4000 px at 3000x4000 -> 240x320) they are read from
// global memory through the read-only cache.  The two variants differ only in where the bytes come from: the same table
// entries are summed in the same order.
constexpr int kRealRowsPerCta = 16;
constexpr size_t kRealPrepSmemMax = 227 * 1024;

template <bool STAGED>
__global__ void __launch_bounds__(256) real_prep_kernel(const uint8_t* __restrict__ I, const uint8_t* __restrict__ Ip,
                                                        const float* __restrict__ luts, const int32_t* __restrict__ tab,
                                                        int max_rows, int FH, int FW, int Hh, int W, float* __restrict__ oI,
                                                        float* __restrict__ oIp, float* __restrict__ oIa, float* __restrict__ oIpa) {
  extern __shared__ __align__(16) unsigned char smem[];
  float* lut = reinterpret_cast<float*>(smem);                         // [4][256][3]
  uint8_t* rows = smem + 4 * 768 * sizeof(float);                      // [max_rows][2][FW*3]
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < 4 * 768; i += blockDim.x) lut[i] = luts[(size_t)b * 4 * 768 + i];
  float* outs[4] = {oI, oIp, oIa, oIpa};
  const uint8_t* srcs[2] = {I + (size_t)b * FH * FW * 3, Ip + (size_t)b * FH * FW * 3};
  const int rowlen = W * 3, dy0 = blockIdx.x * kRealRowsPerCta, dy1 = min(dy0 + kRealRowsPerCta, Hh);
  if (!tab) {                                                          // full size == network size: a table lookup
    __syncthreads();
    for (int o = dy0 * rowlen + threadIdx.x; o < dy1 * rowlen; o += blockDim.x) {
      const int c = o % 3;
      const size_t e = (size_t)b * Hh * rowlen + o;
#pragma unroll
      for (int t = 0; t < 4; ++t) outs[t][e] = lut[t * 768 + srcs[t & 1][o] * 3 + c];
    }
    return;
  }
  const int nx = tab[0], ny = tab[1];
  const int32_t* xofs = tab + 2;
  const int32_t* xsrc = xofs + W + 1;
  const float* xw = reinterpret_cast<const float*>(xsrc + nx);
  const int32_t* yofs = xsrc + 2 * nx;
  const int32_t* ysrc = yofs + Hh + 1;
  const float* yw = reinterpret_cast<const float*>(ysrc + ny);
  const int srclen = FW * 3;
  for (int dy = dy0; dy < dy1; ++dy) {
    const int k0 = yofs[dy], nk = yofs[dy + 1] - k0;
    __syncthreads();                                                   // previous row's readers are done (and the tables)
    if (STAGED) {
      for (int i = threadIdx.x; i < nk * 2 * srclen; i += blockDim.x) {
        const int k = i / (2 * srclen), r = i - k * 2 * srclen, im = r / srclen, x = r - im * srclen;
        rows[(k * 2 + im) * srclen + x] = (im ? srcs[1] : srcs[0])[(size_t)ysrc[k0 + k] * srclen + x];
      }
      __syncthreads();
    }
    // byte s of source row k (of this output row) of image im
    auto src_at = [&](int k, int im, int s) -> int {
      if (STAGED) return rows[(k * 2 + im) * srclen + s];
      return __ldg(srcs[im] + (size_t)ysrc[k0 + k] * srclen + s);
    };
    for (int o = threadIdx.x; o < rowlen; o += blockDim.x) {
      const int dx = o / 3, c = o - dx * 3, j0 = xofs[dx], j1 = xofs[dx + 1];
      float sum[4];
      for (int k = 0; k < nk; ++k) {
        const float beta = yw[k0 + k];
        float buf[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        for (int j = j0; j < j1; ++j) {
          const float alpha = xw[j];
          const int s = xsrc[j] * 3 + c;
#pragma unroll
          for (int t = 0; t < 4; ++t)
            buf[t] = __fadd_rn(buf[t], __fmul_rn(lut[t * 768 + src_at(k, t & 1, s) * 3 + c], alpha));
        }
#pragma unroll
        for (int t = 0; t < 4; ++t) sum[t] = k == 0 ? __fmul_rn(beta, buf[t]) : __fadd_rn(sum[t], __fmul_rn(beta, buf[t]));
      }
      const size_t e = ((size_t)b * Hh + dy) * rowlen + o;
#pragma unroll
      for (int t = 0; t < 4; ++t) outs[t][e] = sum[t];
    }
  }
}

// ---- the real harness's metric --------------------------------------------------------------------------------------------
__device__ __forceinline__ float pairwise8_f32(const float* s) {       // NumPy's pairwise sum of 8 values
  return __fadd_rn(__fadd_rn(__fadd_rn(s[0], s[1]), __fadd_rn(s[2], s[3])), __fadd_rn(__fadd_rn(s[4], s[5]), __fadd_rn(s[6], s[7])));
}
__device__ __forceinline__ double pairwise8_f64(const double* s) {
  return __dadd_rn(__dadd_rn(__dadd_rn(s[0], s[1]), __dadd_rn(s[2], s[3])), __dadd_rn(__dadd_rn(s[4], s[5]), __dadd_rn(s[6], s[7])));
}

__global__ void ecc_corr_h4p_kernel(const float* __restrict__ Wm, const int32_t* __restrict__ status, const float* __restrict__ gt,
                                    float* __restrict__ pred, double* __restrict__ h_loss, int32_t* __restrict__ fail, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float c1[8], c2[8], p[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {                                        // clicked on 480x640 frames: / 2 onto 240x320
    c1[k] = __fdiv_rn(gt[(size_t)b * 16 + k], 2.0f);
    c2[k] = __fdiv_rn(gt[(size_t)b * 16 + 8 + k], 2.0f);
  }
  if (status[b] != 0) {                                                // cv2 raised: pred = float64 zeros, no identity bound
    double s[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const double d = __dsub_rn((double)c1[k], (double)c2[k]);
      s[k] = __dmul_rn(d, d);
      pred[(size_t)b * 8 + k] = 0.0f;
    }
    h_loss[b] = __dsqrt_rn(__ddiv_rn(pairwise8_f64(s), 8.0));
    fail[b] = 1;
    return;
  }
  double m[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) m[k] = (double)Wm[(size_t)b * 9 + k];
#pragma unroll
  for (int k = 0; k < 4; ++k) {                                        // cv2.perspectiveTransform on fp32 points, W not inverted
    const double x = c1[2 * k], y = c1[2 * k + 1];
    double w = __dadd_rn(__dadd_rn(__dmul_rn(x, m[6]), __dmul_rn(y, m[7])), m[8]);
    float X = 0.0f, Y = 0.0f;
    if (fabs(w) > (double)FLT_EPSILON) {
      w = __ddiv_rn(1.0, w);
      X = (float)__dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, m[0]), __dmul_rn(y, m[1])), m[2]), w);
      Y = (float)__dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, m[3]), __dmul_rn(y, m[4])), m[5]), w);
    }
    p[2 * k] = __fsub_rn(X, c1[2 * k]);
    p[2 * k + 1] = __fsub_rn(Y, c1[2 * k + 1]);
  }
  float se[8], si[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (p[k] >= 80.0f) p[k] = 80.0f;
    if (p[k] <= -80.0f) p[k] = -80.0f;
    pred[(size_t)b * 8 + k] = p[k];
    const float d = __fsub_rn(__fadd_rn(p[k], c1[k]), c2[k]), di = __fsub_rn(c1[k], c2[k]);
    se[k] = __fmul_rn(d, d);
    si[k] = __fmul_rn(di, di);
  }
  float h = __fsqrt_rn(__fdiv_rn(pairwise8_f32(se), 8.0f));
  const float ident = __fsqrt_rn(__fdiv_rn(pairwise8_f32(si), 8.0f));
  int f = 0;
  if (ident < h) { f = 2; h = ident; }
  h_loss[b] = (double)h;
  fail[b] = f;
}

}  // namespace udh

using namespace udh;

extern "C" int udh_resize_area_up_u8(const uint8_t* src, const int32_t* tab, uint8_t* dst, int n, int src_h, int src_w, int dst_h,
                                     int dst_w, void* stream) {
  UDH_REQUIRE(src && tab && dst, "udh_resize_area_up_u8: null pointer");
  UDH_REQUIRE(n >= 0 && src_h >= 1 && src_w >= 1 && dst_h > src_h && dst_w > src_w, "udh_resize_area_up_u8: bad dimensions");
  if (n == 0) return UDH_OK;
  cudaStream_t st = as_stream(stream);
  ProfScope ps(PROF_ELTWISE, st);
  resize_up_u8_kernel<false><<<dim3((dst_h * dst_w + 255) / 256, n), 256, 0, st>>>(src, tab, dst, src_h, src_w, dst_h, dst_w);
  return check_launch("udh_resize_area_up_u8");
}

extern "C" int udh_resize_linear_u8(const uint8_t* src, const int32_t* tab, uint8_t* dst, int n, int src_h, int src_w, int dst_h,
                                    int dst_w, void* stream) {
  UDH_REQUIRE(src && tab && dst, "udh_resize_linear_u8: null pointer");
  UDH_REQUIRE(n >= 0 && src_h >= 1 && src_w >= 1 && dst_h >= 1 && dst_w >= 1 && (int64_t)dst_h * dst_w < INT32_MAX,
              "udh_resize_linear_u8: bad dimensions");
  if (n == 0) return UDH_OK;
  cudaStream_t st = as_stream(stream);
  ProfScope ps(PROF_ELTWISE, st);
  resize_up_u8_kernel<true><<<dim3((dst_h * dst_w + 255) / 256, n), 256, 0, st>>>(src, tab, dst, src_h, src_w, dst_h, dst_w);
  return check_launch("udh_resize_linear_u8");
}

extern "C" size_t udh_real_prep_smem_bytes(int max_rows, int full_w) {
  return (size_t)4 * 768 * sizeof(float) + (size_t)max_rows * 2 * full_w * 3;
}

extern "C" int udh_real_prep(const uint8_t* I, const uint8_t* I_prime, const float* luts, const int32_t* tab, int max_rows, int B,
                             int full_h, int full_w, int img_h, int img_w, float* I_plain, float* I_prime_plain, float* I_aug,
                             float* I_prime_aug, void* stream) {
  UDH_REQUIRE(I && I_prime && luts && I_plain && I_prime_plain && I_aug && I_prime_aug, "udh_real_prep: null pointer");
  UDH_REQUIRE(B >= 1 && img_h >= 1 && img_w >= 1 && full_h >= img_h && full_w >= img_w, "udh_real_prep: bad dimensions");
  UDH_REQUIRE(tab || (full_h == img_h && full_w == img_w), "udh_real_prep: a resize needs the area tables");
  UDH_REQUIRE(!tab || max_rows >= 1, "udh_real_prep: max_rows must be >= 1");
  const bool staged = udh_real_prep_smem_bytes(tab ? max_rows : 0, full_w) <= kRealPrepSmemMax;
  const size_t smem = udh_real_prep_smem_bytes(staged && tab ? max_rows : 0, full_w);
  cudaStream_t st = as_stream(stream);
  ProfScope ps(PROF_ELTWISE, st);
  auto kern = staged ? real_prep_kernel<true> : real_prep_kernel<false>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      set_error("udh_real_prep: %s", cudaGetErrorString(e));
      return UDH_ECUDA;
    }
  }
  kern<<<dim3((img_h + kRealRowsPerCta - 1) / kRealRowsPerCta, B), 256, smem, st>>>(
      I, I_prime, luts, tab, max_rows, full_h, full_w, img_h, img_w, I_plain, I_prime_plain, I_aug, I_prime_aug);
  return check_launch("udh_real_prep");
}

extern "C" int udh_ecc_corr_h4p(const float* W, const int32_t* status, const float* gt, float* pred_h4p, double* h_loss, int32_t* fail,
                                int B, void* stream) {
  UDH_REQUIRE(W && status && gt && pred_h4p && h_loss && fail, "udh_ecc_corr_h4p: null pointer");
  UDH_REQUIRE(B >= 0, "udh_ecc_corr_h4p: negative batch");
  if (B == 0) return UDH_OK;
  ecc_corr_h4p_kernel<<<(B + 127) / 128, 128, 0, as_stream(stream)>>>(W, status, gt, pred_h4p, h_loss, fail, B);
  return check_launch("udh_ecc_corr_h4p");
}
