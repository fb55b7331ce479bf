// fp32 CUDA-core building blocks of the 4-point regressor (Row C; code/homography_model.py:88-133).
// This is the PARITY numeric mode (UDH_NUMERIC_FP32): fp32 FFMA implicit-GEMM convolutions, max-pool, SGEMM for
// the two fully connected layers, dropout, and their backward passes.  The throughput mode (bf16 wgmma) is in
// conv_tc.cu and is validated against these kernels.
#include "cnn_kernels.cuh"

namespace udh {

namespace {
inline unsigned grid1d(size_t want, size_t cap) { return (unsigned)(want < cap ? (want ? want : 1) : cap); }
constexpr int TH = 8, TW = 16;          // output tile (rows x cols) of the conv / wgrad kernels
constexpr int PITCH = 20;               // smem column pitch of the (TW+2)-wide halo rows (16-byte aligned windows)
constexpr int PLANE = (TH + 2) * PITCH; // floats per channel plane

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__device__ __forceinline__ uint8_t keep_bit(uint64_t seed, uint64_t salt, uint64_t idx) {
  return (uint8_t)(splitmix64(seed ^ splitmix64(salt) ^ (idx * 0xD1342543DE82EF95ull)) >> 63);
}

// Stage a (TH+2) x (TW+2) x CK halo tile of an NHWC image into smem as [CK][TH+2][PITCH] (zero padded).
template <int CK, bool TWO_PLANE>
__device__ __forceinline__ void load_halo(float* in_s, const float* __restrict__ in0, const float* __restrict__ in1,
                                          int n, int y0, int x0, int H, int W, int Cin, int ci0) {
  constexpr int NPIX = (TH + 2) * (TW + 2);
  if (TWO_PLANE) {
    for (int it = threadIdx.x; it < NPIX * 2; it += blockDim.x) {
      const int c = it / NPIX, p = it - c * NPIX;
      const int r = p / (TW + 2), cc = p - r * (TW + 2);
      const int gy = y0 - 1 + r, gx = x0 - 1 + cc;
      float v = 0.f;
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = __ldg((c == 0 ? in0 : in1) + ((size_t)n * H + gy) * W + gx);
      in_s[c * PLANE + r * PITCH + cc] = v;
    }
  } else {
    constexpr int Q = CK >= 4 ? CK / 4 : 1;
    for (int it = threadIdx.x; it < NPIX * Q; it += blockDim.x) {
      const int p = it / Q, q = it - p * Q;
      const int r = p / (TW + 2), cc = p - r * (TW + 2);
      const int gy = y0 - 1 + r, gx = x0 - 1 + cc;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gy >= 0 && gy < H && gx >= 0 && gx < W)
        v = __ldg(reinterpret_cast<const float4*>(in0 + (((size_t)n * H + gy) * W + gx) * Cin + ci0 + q * 4));
      float* d = in_s + (q * 4) * PLANE + r * PITCH + cc;
      d[0] = v.x; d[PLANE] = v.y; d[2 * PLANE] = v.z; d[3 * PLANE] = v.w;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// conv 3x3, pad 1, stride 1: CTA = 8x16 output pixels x 64 output channels, thread = 8 pixels x 4 channels.
// ---------------------------------------------------------------------------------------------------------
template <int CK, bool TWO_PLANE>
__global__ void __launch_bounds__(256) conv3x3_kernel(const float* __restrict__ in0, const float* __restrict__ in1,
                                                      const float* __restrict__ w, const float* __restrict__ bias,
                                                      const float* __restrict__ mask_src, float* __restrict__ out, int H,
                                                      int W, int Cin, int Cout, int relu) {
  __shared__ __align__(16) float in_s[CK * PLANE];
  __shared__ __align__(16) float w_s[9 * CK * 64];
  const int tiles_x = W / TW;
  const int ty = blockIdx.x / tiles_x, tx = blockIdx.x - ty * tiles_x;
  const int n = blockIdx.y, co0 = blockIdx.z * 64;
  const int y0 = ty * TH, x0 = tx * TW;
  const int cg = threadIdx.x & 15, pg = threadIdx.x >> 4;
  const int row = pg >> 1, col0 = (pg & 1) * 8;

  float acc[8][4];
#pragma unroll
  for (int p = 0; p < 8; ++p)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[p][j] = 0.f;

  for (int ci0 = 0; ci0 < Cin; ci0 += CK) {
    __syncthreads();
    load_halo<CK, TWO_PLANE>(in_s, in0, in1, n, y0, x0, H, W, Cin, ci0);
    for (int it = threadIdx.x; it < 9 * CK * 16; it += 256) {
      const int rowi = it >> 4, f4 = it & 15;
      const int tap = rowi / CK, c = rowi - tap * CK;
      *reinterpret_cast<float4*>(w_s + rowi * 64 + f4 * 4) =
          __ldg(reinterpret_cast<const float4*>(w + ((size_t)(tap * Cin + ci0 + c)) * Cout + co0 + f4 * 4));
    }
    __syncthreads();
#pragma unroll 2
    for (int c = 0; c < CK; ++c) {
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        const float* ip = in_s + c * PLANE + (row + ky) * PITCH + col0;
        const float4 a0 = *reinterpret_cast<const float4*>(ip);
        const float4 a1 = *reinterpret_cast<const float4*>(ip + 4);
        const float2 a2 = *reinterpret_cast<const float2*>(ip + 8);
        const float a[10] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y};
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const float4 wv = *reinterpret_cast<const float4*>(w_s + ((ky * 3 + kx) * CK + c) * 64 + cg * 4);
#pragma unroll
          for (int p = 0; p < 8; ++p) {
            acc[p][0] = fmaf(a[p + kx], wv.x, acc[p][0]);
            acc[p][1] = fmaf(a[p + kx], wv.y, acc[p][1]);
            acc[p][2] = fmaf(a[p + kx], wv.z, acc[p][2]);
            acc[p][3] = fmaf(a[p + kx], wv.w, acc[p][3]);
          }
        }
      }
    }
  }
  float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
  if (bias) bv = __ldg(reinterpret_cast<const float4*>(bias + co0 + cg * 4));
  const int y = y0 + row;
#pragma unroll
  for (int p = 0; p < 8; ++p) {
    const size_t o = (((size_t)n * H + y) * W + x0 + col0 + p) * Cout + co0 + cg * 4;
    float4 v = make_float4(acc[p][0] + bv.x, acc[p][1] + bv.y, acc[p][2] + bv.z, acc[p][3] + bv.w);
    if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    if (mask_src) {
      const float4 m = __ldg(reinterpret_cast<const float4*>(mask_src + o));
      v.x = m.x > 0.f ? v.x : 0.f; v.y = m.y > 0.f ? v.y : 0.f; v.z = m.z > 0.f ? v.z : 0.f; v.w = m.w > 0.f ? v.w : 0.f;
    }
    *reinterpret_cast<float4*>(out + o) = v;
  }
}

// ---------------------------------------------------------------------------------------------------------
// weight gradient: CTA = (range of 8x16 pixel tiles) x CK input channels x 64 output channels,
// thread = 1 input channel x 4 output channels x 9 taps; pixels are the reduction dimension.
// ---------------------------------------------------------------------------------------------------------
template <int CK, bool TWO_PLANE>
__global__ void __launch_bounds__(256) wgrad3x3_kernel(const float* __restrict__ x0p, const float* __restrict__ x1p,
                                                       const float* __restrict__ g, float* __restrict__ dW,
                                                       float* __restrict__ db, int B, int H, int W, int Cin, int Cout,
                                                       int tiles_per_cta) {
  constexpr int SPLIT = 256 / (CK * 16);
  __shared__ __align__(16) float x_s[CK * PLANE];
  __shared__ __align__(16) float g_s[TH * TW * 64];
  const int ci0 = blockIdx.y * CK, co0 = blockIdx.z * 64;
  const int cg = threadIdx.x & 15;
  const int ci = (threadIdx.x >> 4) % CK, s = (threadIdx.x >> 4) / CK;
  const int tiles_x = W / TW, tiles_img = tiles_x * (H / TH);
  const int t_begin = blockIdx.x * tiles_per_cta;
  const int t_end = min(t_begin + tiles_per_cta, B * tiles_img);

  float acc[9][4], bacc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[t][j] = 0.f;

  for (int t = t_begin; t < t_end; ++t) {
    const int n = t / tiles_img, tt = t - n * tiles_img;
    const int ty = tt / tiles_x, tx = tt - ty * tiles_x;
    const int y0 = ty * TH, x0 = tx * TW;
    __syncthreads();
    load_halo<CK, TWO_PLANE>(x_s, x0p, x1p, n, y0, x0, H, W, Cin, ci0);
    for (int it = threadIdx.x; it < TH * TW * 16; it += 256) {
      const int p = it >> 4, f4 = it & 15;
      const int r = p >> 4, c = p & 15;
      *reinterpret_cast<float4*>(g_s + p * 64 + f4 * 4) =
          __ldg(reinterpret_cast<const float4*>(g + (((size_t)n * H + y0 + r) * W + x0 + c) * Cout + co0 + f4 * 4));
    }
    __syncthreads();
    for (int r = s; r < TH; r += SPLIT) {
      float xw[3][3];
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        xw[ky][0] = x_s[ci * PLANE + (r + ky) * PITCH + 0];
        xw[ky][1] = x_s[ci * PLANE + (r + ky) * PITCH + 1];
      }
#pragma unroll
      for (int c = 0; c < TW; ++c) {
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) xw[ky][2] = x_s[ci * PLANE + (r + ky) * PITCH + c + 2];
        const float4 gv = *reinterpret_cast<const float4*>(g_s + (r * TW + c) * 64 + cg * 4);
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            acc[ky * 3 + kx][0] = fmaf(xw[ky][kx], gv.x, acc[ky * 3 + kx][0]);
            acc[ky * 3 + kx][1] = fmaf(xw[ky][kx], gv.y, acc[ky * 3 + kx][1]);
            acc[ky * 3 + kx][2] = fmaf(xw[ky][kx], gv.z, acc[ky * 3 + kx][2]);
            acc[ky * 3 + kx][3] = fmaf(xw[ky][kx], gv.w, acc[ky * 3 + kx][3]);
          }
        bacc[0] += gv.x; bacc[1] += gv.y; bacc[2] += gv.z; bacc[3] += gv.w;
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) { xw[ky][0] = xw[ky][1]; xw[ky][1] = xw[ky][2]; }
      }
    }
  }
  if (t_begin < t_end) {
#pragma unroll
    for (int t = 0; t < 9; ++t)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        atomicAdd(dW + ((size_t)(t * Cin + ci0 + ci)) * Cout + co0 + cg * 4 + j, acc[t][j]);
    if (db && blockIdx.y == 0 && ci == 0) {
#pragma unroll
      for (int j = 0; j < 4; ++j) atomicAdd(db + co0 + cg * 4 + j, bacc[j]);
    }
  }
}

__global__ void rotate_weights_kernel(const float* __restrict__ w, float* __restrict__ wrot, int Cin, int Cout) {
  const int total = 9 * Cin * Cout;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    // i indexes wrot[tap][co][ci]
    const int ci = i % Cin, co = (i / Cin) % Cout, tap = i / (Cin * Cout);
    wrot[i] = w[((size_t)((8 - tap) * Cin + ci)) * Cout + co];
  }
}

__global__ void maxpool_fwd_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W, int C) {
  const int C4 = C >> 2, OH = H >> 1, OW = W >> 1;
  const size_t total = (size_t)B * OH * OW * C4;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = i % C4;
    size_t r = i / C4;
    const int ox = r % OW; r /= OW;
    const int oy = r % OH;
    const int n = r / OH;
    const float4* p = reinterpret_cast<const float4*>(in + (((size_t)n * H + 2 * oy) * W + 2 * ox) * C) + c4;
    const float4 a = __ldg(p), b = __ldg(p + C4), c = __ldg(p + (size_t)W * C4), d = __ldg(p + (size_t)W * C4 + C4);
    float4 m;
    m.x = fmaxf(fmaxf(a.x, b.x), fmaxf(c.x, d.x));
    m.y = fmaxf(fmaxf(a.y, b.y), fmaxf(c.y, d.y));
    m.z = fmaxf(fmaxf(a.z, b.z), fmaxf(c.z, d.z));
    m.w = fmaxf(fmaxf(a.w, b.w), fmaxf(c.w, d.w));
    reinterpret_cast<float4*>(out)[i] = m;
  }
}

__device__ __forceinline__ void route1(float a, float b, float c, float d, float g, float& oa, float& ob, float& oc, float& od) {
  // first arg-max in window scan order (row-major), gradient only where the winner is > 0 (ReLU of the producer)
  float m = a; int k = 0;
  if (b > m) { m = b; k = 1; }
  if (c > m) { m = c; k = 2; }
  if (d > m) { m = d; k = 3; }
  const float v = m > 0.f ? g : 0.f;
  oa = k == 0 ? v : 0.f; ob = k == 1 ? v : 0.f; oc = k == 2 ? v : 0.f; od = k == 3 ? v : 0.f;
}

__global__ void maxpool_bwd_kernel(const float* __restrict__ in, const float* __restrict__ dout, float* __restrict__ din,
                                   int B, int H, int W, int C) {
  const int C4 = C >> 2, OH = H >> 1, OW = W >> 1;
  const size_t total = (size_t)B * OH * OW * C4;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = i % C4;
    size_t r = i / C4;
    const int ox = r % OW; r /= OW;
    const int oy = r % OH;
    const int n = r / OH;
    const size_t base = (((size_t)n * H + 2 * oy) * W + 2 * ox) * C;
    const float4* p = reinterpret_cast<const float4*>(in + base) + c4;
    const float4 a = __ldg(p), b = __ldg(p + C4), c = __ldg(p + (size_t)W * C4), d = __ldg(p + (size_t)W * C4 + C4);
    const float4 g = __ldg(reinterpret_cast<const float4*>(dout) + i);
    float4 oa, ob, oc, od;
    route1(a.x, b.x, c.x, d.x, g.x, oa.x, ob.x, oc.x, od.x);
    route1(a.y, b.y, c.y, d.y, g.y, oa.y, ob.y, oc.y, od.y);
    route1(a.z, b.z, c.z, d.z, g.z, oa.z, ob.z, oc.z, od.z);
    route1(a.w, b.w, c.w, d.w, g.w, oa.w, ob.w, oc.w, od.w);
    float4* q = reinterpret_cast<float4*>(din + base) + c4;
    q[0] = oa; q[C4] = ob; q[(size_t)W * C4] = oc; q[(size_t)W * C4 + C4] = od;
  }
}

// ---------------------------------------------------------------------------------------------------------
// SGEMM with explicit strides, 64x64x16 tiles, 4x4 micro-tiles, optional split-K (atomic accumulation).
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sgemm_kernel(const float* __restrict__ A, int64_t a_rs, int64_t a_cs,
                                                    const float* __restrict__ Bm, int64_t b_rs, int64_t b_cs,
                                                    float* __restrict__ C, int64_t ldc, int M, int N, int K, int k_chunk,
                                                    int atomic, float* __restrict__ slab) {
  pdl_wait(); pdl_trigger();   // launched through launch_chain (common.cuh)
  __shared__ __align__(16) float As[16][68];
  __shared__ __align__(16) float Bs[16][68];
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int k_begin = blockIdx.z * k_chunk, k_end = min(K, k_begin + k_chunk);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = k_begin; k0 < k_end; k0 += 16) {
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int idx = threadIdx.x + e * 256;
      int m, k;
      if (a_cs == 1) { m = idx >> 4; k = idx & 15; } else { k = idx >> 6; m = idx & 63; }
      float v = 0.f;
      if (m0 + m < M && k0 + k < k_end) v = __ldg(A + (int64_t)(m0 + m) * a_rs + (int64_t)(k0 + k) * a_cs);
      As[k][m] = v;
      int kk, nn;
      if (b_cs == 1) { kk = idx >> 6; nn = idx & 63; } else { nn = idx >> 4; kk = idx & 15; }
      float u = 0.f;
      if (n0 + nn < N && k0 + kk < k_end) u = __ldg(Bm + (int64_t)(k0 + kk) * b_rs + (int64_t)(n0 + nn) * b_cs);
      Bs[kk][nn] = u;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
  }
  // split-K: each split stores its partial product in its own slab ([split][M][N]); the launcher adds them in split order
  float* part = slab ? slab + (size_t)blockIdx.z * M * N : nullptr;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      if (part) { part[(size_t)m * N + n] = acc[i][j]; continue; }
      float* dst = C + (int64_t)m * ldc + n;
      if (atomic) atomicAdd(dst, acc[i][j]); else *dst = acc[i][j];
    }
  }
}

__global__ void bias_act_dropout_kernel(const float* __restrict__ x, const float* __restrict__ bias, float* __restrict__ act,
                                        float* __restrict__ drop, uint8_t* __restrict__ mask, int rows, int cols, int relu,
                                        int gen_mask, uint64_t seed, uint64_t salt) {
  pdl_wait(); pdl_trigger();   // launched through launch_chain (common.cuh)
  const size_t total = (size_t)rows * cols;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    float v = x[i] + (bias ? __ldg(bias + (i % cols)) : 0.f);
    if (relu) v = fmaxf(v, 0.f);
    if (act) act[i] = v;
    if (drop) {
      float d = v;
      if (mask) {
        uint8_t k = gen_mask ? keep_bit(seed, salt, i) : mask[i];
        if (gen_mask) mask[i] = k;
        d = k ? v * 2.0f : 0.f;                              // slim.dropout keep_prob 0.5: kept values scaled by 1/0.5
      }
      drop[i] = d;
    }
  }
}

__global__ void drop_relu_bwd_kernel(float* __restrict__ g, const uint8_t* __restrict__ mask, const float* __restrict__ act,
                                     size_t n) {
  pdl_wait(); pdl_trigger();   // launched through launch_chain (common.cuh)
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float v = g[i];
    if (mask) v = mask[i] ? v * 2.0f : 0.f;
    g[i] = act[i] > 0.f ? v : 0.f;
  }
}

// partial column sums of the row slices blockIdx.y, one slab each ([slice][cols]); the launcher adds them in slice order
__global__ void colsum_kernel(const float* __restrict__ g, float* __restrict__ part, int rows, int cols) {
  pdl_wait(); pdl_trigger();   // launched through launch_chain (common.cuh)
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  float s = 0.f;
  for (int r = blockIdx.y; r < rows; r += gridDim.y) s += g[(size_t)r * cols + c];
  part[(size_t)blockIdx.y * cols + c] = s;
}

}  // namespace

int conv3x3_simt(const float* in0, const float* in1, const float* w, const float* bias, const float* mask_src,
                 float* out, int B, int H, int W, int Cin, int Cout, int relu, cudaStream_t st) {
  UDH_REQUIRE(H % TH == 0 && W % TW == 0 && Cout % 64 == 0, "conv3x3: unsupported shape H=%d W=%d Cout=%d", H, W, Cout);
  dim3 grid((H / TH) * (W / TW), B, Cout / 64);
  if (in1) {
    UDH_REQUIRE(Cin == 2, "conv3x3: two-plane input needs Cin == 2");
    conv3x3_kernel<2, true><<<grid, 256, 0, st>>>(in0, in1, w, bias, mask_src, out, H, W, Cin, Cout, relu);
  } else {
    UDH_REQUIRE(Cin % 8 == 0, "conv3x3: Cin must be a multiple of 8 (got %d)", Cin);
    conv3x3_kernel<8, false><<<grid, 256, 0, st>>>(in0, nullptr, w, bias, mask_src, out, H, W, Cin, Cout, relu);
  }
  return check_launch("conv3x3_simt");
}

int wgrad3x3_simt(const float* x0, const float* x1, const float* g, float* dW, float* db, int B, int H, int W, int Cin,
                  int Cout, cudaStream_t st) {
  UDH_REQUIRE(H % TH == 0 && W % TW == 0 && Cout % 64 == 0, "wgrad3x3: unsupported shape");
  const int tiles = B * (H / TH) * (W / TW);
  if (x1) {
    UDH_REQUIRE(Cin == 2, "wgrad3x3: two-plane input needs Cin == 2");
    const int ctas = min(tiles, kSmCount * 4 / (Cout / 64));
    const int per = (tiles + ctas - 1) / ctas;
    dim3 grid((tiles + per - 1) / per, 1, Cout / 64);
    wgrad3x3_kernel<2, true><<<grid, 256, 0, st>>>(x0, x1, g, dW, db, B, H, W, Cin, Cout, per);
  } else {
    UDH_REQUIRE(Cin % 16 == 0, "wgrad3x3: Cin must be a multiple of 16 (got %d)", Cin);
    const int groups = (Cin / 16) * (Cout / 64);
    const int ctas = max(1, min(tiles, (kSmCount * 4 + groups - 1) / groups));
    const int per = (tiles + ctas - 1) / ctas;
    dim3 grid((tiles + per - 1) / per, Cin / 16, Cout / 64);
    wgrad3x3_kernel<16, false><<<grid, 256, 0, st>>>(x0, nullptr, g, dW, db, B, H, W, Cin, Cout, per);
  }
  return check_launch("wgrad3x3_simt");
}

int rotate_weights(const float* w, float* wrot, int Cin, int Cout, cudaStream_t st) {
  const int total = 9 * Cin * Cout;
  rotate_weights_kernel<<<(total + 255) / 256, 256, 0, st>>>(w, wrot, Cin, Cout);
  return check_launch("rotate_weights");
}

int maxpool2x2_fwd(const float* in, float* out, int B, int H, int W, int C, cudaStream_t st) {
  UDH_REQUIRE(H % 2 == 0 && W % 2 == 0 && C % 4 == 0, "maxpool: unsupported shape");
  const size_t total = (size_t)B * (H / 2) * (W / 2) * (C / 4);
  maxpool_fwd_kernel<<<grid1d((total + 255) / 256, kSmCount * 32), 256, 0, st>>>(in, out, B, H, W, C);
  return check_launch("maxpool2x2_fwd");
}

int maxpool2x2_bwd(const float* in, const float* dout, float* din, int B, int H, int W, int C, cudaStream_t st) {
  UDH_REQUIRE(H % 2 == 0 && W % 2 == 0 && C % 4 == 0, "maxpool: unsupported shape");
  const size_t total = (size_t)B * (H / 2) * (W / 2) * (C / 4);
  maxpool_bwd_kernel<<<grid1d((total + 255) / 256, kSmCount * 32), 256, 0, st>>>(in, dout, din, B, H, W, C);
  return check_launch("maxpool2x2_bwd");
}

int sgemm_simt(const float* A, int64_t a_rs, int64_t a_cs, const float* Bm, int64_t b_rs, int64_t b_cs, float* C,
               int64_t ldc, int M, int N, int K, int split_k, int accumulate, cudaStream_t st) {
  UDH_REQUIRE(M > 0 && N > 0 && K > 0 && split_k >= 1, "sgemm: bad dimensions");
  int k_chunk = ((K + split_k - 1) / split_k + 15) / 16 * 16;
  split_k = (K + k_chunk - 1) / k_chunk;
  dim3 grid((N + 63) / 64, (M + 63) / 64, split_k);
  float* slab = nullptr;
  if (split_k > 1) {
    UDH_REQUIRE(ldc == N, "sgemm: split-K needs a dense output (ldc %lld, N %d)", (long long)ldc, N);
    slab = slab_scratch((size_t)split_k * M * N, st);
    if (!slab) return UDH_ECUDA;
  }
  launch_chain(sgemm_kernel, grid, dim3(256), 0, st, A, a_rs, a_cs, Bm, b_rs, b_cs, C, ldc, M, N, K, k_chunk,
               accumulate ? 1 : 0, slab);
  if (int rc = check_launch("sgemm_simt")) return rc;
  if (!slab) return UDH_OK;
  SlabSegments t;
  t.count = 1;
  t.s[0] = SlabSegment{slab, C, (size_t)M * N, split_k, M * N};
  return slab_reduce(t, st);
}

int bias_act_dropout(const float* x, const float* bias, float* act, float* drop, uint8_t* mask, int rows, int cols,
                     int relu, int gen_mask, uint64_t seed, uint64_t salt, cudaStream_t st) {
  const size_t total = (size_t)rows * cols;
  launch_chain(bias_act_dropout_kernel, dim3(grid1d((total + 255) / 256, kSmCount * 16)), dim3(256), 0, st,
               x, bias, act, drop, mask, rows, cols, relu, gen_mask, seed, salt);
  return check_launch("bias_act_dropout");
}

int dropout_fwd(const float* x, float* drop, uint8_t* mask, size_t n, uint64_t seed, uint64_t salt, cudaStream_t st) {
  return bias_act_dropout(x, nullptr, nullptr, drop, mask, 1, (int)n, 0, 1, seed, salt, st);
}

int drop_relu_bwd(float* g, const uint8_t* mask, const float* act, size_t n, cudaStream_t st) {
  launch_chain(drop_relu_bwd_kernel, dim3(grid1d((n + 255) / 256, kSmCount * 16)), dim3(256), 0, st, g, mask, act, n);
  return check_launch("drop_relu_bwd");
}

int colsum_accum(const float* g, float* db, int rows, int cols, cudaStream_t st) {
  dim3 grid((cols + 127) / 128, min(rows, 16));
  float* part = slab_scratch((size_t)grid.y * cols, st);
  if (!part) return UDH_ECUDA;
  launch_chain(colsum_kernel, grid, dim3(128), 0, st, g, part, rows, cols);
  if (int rc = check_launch("colsum_accum")) return rc;
  SlabSegments t;
  t.count = 1;
  t.s[0] = SlabSegment{part, db, (size_t)cols, (int)grid.y, cols};
  return slab_reduce(t, st);
}

}  // namespace udh
