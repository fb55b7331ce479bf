// conv1_1 (2 -> 64 channels) on wgmma for the bf16 mode.  K = 3*3*2 = 18 is far below one 64-wide k-block, so the layer
// is bound by its 277 MB bf16 output (forward) / gradient input (wgrad), not by math; the point of using the tensor pipe
// is to get the 2.4 GMAC off the CUDA cores.  Both kernels build an explicit im2col tile in shared memory:
//   A[128 pixels of one image row][64] bf16, k = tap*2 + plane for k < 18 (k = 18 is a constant 1 for the wgrad's bias
//   row), zero beyond — written by the CTA's 128 threads (one warpgroup, thread = pixel) in the SWIZZLE_128B pattern the
//   MMA expects; the same warpgroup then issues the MMAs and drains the accumulators.
// forward : D[pixel][co] = A . W^T   (A K-major, W [64 co][64 k] K-major, two M = 64 halves, N = 64), epilogue = bias +
//           ReLU + bf16 pack + 1-bit ReLU mask + TMA store into the zero-bordered stream.  Several CTAs share an SM, so
//           one CTA's MMAs overlap another's im2col build and epilogue.
// wgrad   : D[k][co] += A^T . G      (the same A bytes read as an MN-major operand, M = 64; G row block by TMA;
//           K = 128 pixels per tile, 8 k-steps), accumulated in registers over the CTA's whole run; row 18 is the bias
//           gradient.
#pragma once
#include "tc_common.cuh"

namespace udh {
namespace tc {

struct Conv1Geom { int B, H, W, tiles; };   // tiles = B*H*(W/128) row segments of 128 pixels

// im2col row of pixel (n, y, x): 18 taps -> bf16, written as 3 swizzled 16-byte chunks of row `r` of `tile`
__device__ __forceinline__ void build_im2col_row(uint8_t* tile, int r, const float* __restrict__ I1, const float* __restrict__ I2,
                                                 int n, int y, int x, int H, int W, bool ones_col) {
  float v[24];
#pragma unroll
  for (int i = 0; i < 24; ++i) v[i] = 0.f;
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int gy = y + ky - 1;
    const bool rowok = gy >= 0 && gy < H;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int gx = x + kx - 1;
      if (rowok && gx >= 0 && gx < W) {
        const size_t o = ((size_t)n * H + gy) * W + gx;
        v[(ky * 3 + kx) * 2] = __ldg(I1 + o);
        v[(ky * 3 + kx) * 2 + 1] = __ldg(I2 + o);
      }
    }
  }
  if (ones_col) v[18] = 1.0f;
  const uint32_t rowaddr = smem_u32(tile) + r * 128;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    uint32_t w[4];
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      __nv_bfloat162 p = __floats2bfloat162_rn(v[c * 8 + 2 * h], v[c * 8 + 2 * h + 1]);
      w[h] = *reinterpret_cast<uint32_t*>(&p);
    }
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(rowaddr + (uint32_t)((c ^ (r & 7)) << 4)), "r"(w[0]), "r"(w[1]),
                 "r"(w[2]), "r"(w[3]) : "memory");
  }
}

// ------------------------------------------------------------------------------------------------------------- forward
// 128 threads (thread = pixel = accumulator row).  The CTA is instruction-bound (im2col build + 64-channel epilogue per
// pixel), so several CTAs share an SM (kConv1CtasPerSm).
constexpr int kConv1CtasPerSm = 3;
constexpr size_t kConv1FwdSmem = 1024 + 16384 + 8192 + 16384 + kStgBytes + 256;

// the 128 x 64 accumulator tile held as two M = 64 fragments -> v = row `threadIdx.x` (this thread's pixel), 64 columns
__device__ __forceinline__ void conv1_rows(const float (&a0)[32], const float (&a1)[32], float* stg, float (&v)[2][32]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    __syncthreads();
    stage_acc64(h ? a1 : a0, 0, stg);
    __syncthreads();
    if ((warp >> 1) == h) {
      stg_read32(stg, 32 * (warp & 1) + lane, 0, v[0]);
      stg_read32(stg, 32 * (warp & 1) + lane, 32, v[1]);
    }
  }
}

static __global__ void __launch_bounds__(128, kConv1CtasPerSm)
conv1_tc_fwd_kernel(const __grid_constant__ CUtensorMap tmOut, const Conv1Geom g, const float* __restrict__ I1,
                    const float* __restrict__ I2, const float* __restrict__ w, const float* __restrict__ bias,
                    uint32_t* __restrict__ mask_out) {
  extern __shared__ uint8_t raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sA = base;                       // [128][128 B]
  uint8_t* sW = base + 16384;               // [64 co][128 B]
  uint8_t* sEpi = sW + 8192;                // [4 warps][32][128 B]
  float* sStg = reinterpret_cast<float*>(sEpi + 16384);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // zero the A tile (columns 24..63 stay zero for ever) and build the weight tile W[co][k] = w[tap][ci][co], k = tap*2+ci
  for (int i = threadIdx.x; i < 16384 / 16; i += blockDim.x) reinterpret_cast<uint4*>(sA)[i] = make_uint4(0, 0, 0, 0);
  for (int i = threadIdx.x; i < 64 * 8; i += blockDim.x) {
    const int co = i >> 3, c = i & 7;       // chunk c holds k = 8c .. 8c+7
    uint32_t pk[4];
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const int k0 = c * 8 + 2 * h;
      const float f0 = k0 < 18 ? __ldg(w + k0 * 64 + co) : 0.f, f1 = k0 + 1 < 18 ? __ldg(w + (k0 + 1) * 64 + co) : 0.f;
      __nv_bfloat162 p = __floats2bfloat162_rn(f0, f1);
      pk[h] = *reinterpret_cast<uint32_t*>(&p);
    }
    *reinterpret_cast<uint4*>(sW + co * 128 + ((c ^ (co & 7)) << 4)) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
  }
  if (threadIdx.x == 0) prefetch_tmap(&tmOut);
  pdl_wait();                  // predecessor grid complete (the prologue above touched only parameters, written long before)
  pdl_trigger();
  const int my_tiles = (g.tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int segs = g.W / 128;
  const int px = threadIdx.x;              // pixel within the segment == accumulator row
  uint8_t* stg = sEpi + warp * 4096;
  const uint32_t my_row = smem_u32(stg) + lane * 128;
  const int sw = lane & 7;
  const uint32_t a_lo = desc_lo(smem_u32(sA), 16), w_lo = desc_lo(smem_u32(sW), 16);
  bool store_pending = false;
  for (int i = 0; i < my_tiles; ++i) {
    const int tile = (int)blockIdx.x + i * (int)gridDim.x;
    const int seg = tile % segs, row = tile / segs;
    const int n = row / g.H, y = row - n * g.H;
    // ---- build the im2col tile (the previous tile's MMAs are complete: conv1_rows synchronised after them)
    build_im2col_row(sA, px, I1, I2, n, y, seg * 128 + px, g.H, g.W, false);
    fence_proxy_async();
    __syncthreads();
    float a0[32], a1[32];
    acc_fence(a0); acc_fence(a1);
    wg_fence();
#pragma unroll
    for (int k = 0; k < 2; ++k) {            // k-steps 0,1 cover k = 0..31; everything beyond 18 is zero
      wgmma_bf16<64, 0, 0>(a0, desc_from_lo(a_lo + k * 2), desc_from_lo(w_lo + k * 2), k > 0 ? 1u : 0u);
      wgmma_bf16<64, 0, 0>(a1, desc_from_lo(a_lo + 512 + k * 2), desc_from_lo(w_lo + k * 2), k > 0 ? 1u : 0u);
    }
    wg_commit();
    wg_wait<0>();
    acc_fence(a0); acc_fence(a1);
    // ---- drain
    const int q0w = (n * (g.H + 2) + y + 1) * (g.W + 2) + 1 + seg * 128 + warp * 32;    // padded position of this warp's first pixel
    float vv[2][32];
    conv1_rows(a0, a1, sStg, vv);
    if (store_pending) { if (lane == 0) bulk_wait_read0(); __syncwarp(); store_pending = false; }
    uint32_t mo[2];
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      float (&v)[32] = vv[c];
#pragma unroll
      for (int k = 0; k < 32; k += 4) {
        const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + c * 32 + k));
        v[k] = fmaxf(v[k] + bv.x, 0.f); v[k + 1] = fmaxf(v[k + 1] + bv.y, 0.f);
        v[k + 2] = fmaxf(v[k + 2] + bv.z, 0.f); v[k + 3] = fmaxf(v[k + 3] + bv.w, 0.f);
      }
      uint32_t mw = 0;
#pragma unroll
      for (int k = 0; k < 32; ++k) mw |= (v[k] > 0.f ? 1u : 0u) << k;
      mo[c] = mw;
#pragma unroll
      for (int j4 = 0; j4 < 4; ++j4) {
        __nv_bfloat162 p0 = __floats2bfloat162_rn(v[j4 * 8 + 0], v[j4 * 8 + 1]), p1 = __floats2bfloat162_rn(v[j4 * 8 + 2], v[j4 * 8 + 3]);
        __nv_bfloat162 p2 = __floats2bfloat162_rn(v[j4 * 8 + 4], v[j4 * 8 + 5]), p3 = __floats2bfloat162_rn(v[j4 * 8 + 6], v[j4 * 8 + 7]);
        asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(my_row + (uint32_t)(((c * 4 + j4) ^ sw) << 4)),
                     "r"(*reinterpret_cast<uint32_t*>(&p0)), "r"(*reinterpret_cast<uint32_t*>(&p1)),
                     "r"(*reinterpret_cast<uint32_t*>(&p2)), "r"(*reinterpret_cast<uint32_t*>(&p3)) : "memory");
      }
    }
    if (mask_out) *reinterpret_cast<uint2*>(mask_out + (size_t)(q0w + lane) * 2) = make_uint2(mo[0], mo[1]);
    fence_proxy_async();
    __syncwarp();
    if (lane == 0) { tma_store_2d(&tmOut, stg, 0, q0w); bulk_commit(); }
    store_pending = true;
  }
  if (lane == 0) bulk_wait0();
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------------------- wgrad
// 128 threads build im2col tiles (+ the constant-one column 18) and issue the MMAs; thread 0 loads the G rows by TMA.
constexpr size_t kConv1WgradSmem = 1024 + 2 * 16384 + 256;
constexpr int kConv1SlabFloats = 19 * 64;         // per-CTA partial sums: 18 dW rows + db
static __global__ void __launch_bounds__(128, kConv1CtasPerSm)
conv1_tc_wgrad_kernel(const __grid_constant__ CUtensorMap tmG, const Conv1Geom g, const float* __restrict__ I1,
                      const float* __restrict__ I2, float* __restrict__ slab) {
  extern __shared__ uint8_t raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sA = base;                       // [128][128 B]
  uint8_t* sG = base + 16384;               // [128][128 B]
  uint64_t* g_full = reinterpret_cast<uint64_t*>(sG + 16384);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  for (int i = threadIdx.x; i < 16384 / 16; i += blockDim.x) reinterpret_cast<uint4*>(sA)[i] = make_uint4(0, 0, 0, 0);
  if (threadIdx.x == 0) {
    mbar_init(g_full, 1);
    fence_barrier_init();
    prefetch_tmap(&tmG);
  }
  __syncthreads();
  pdl_wait();                  // predecessor grid complete (the prologue above touched only parameters, written long before)
  pdl_trigger();
  const int my_tiles = (g.tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int segs = g.W / 128;
  const int px = threadIdx.x;
  const uint32_t a_lo = desc_lo(smem_u32(sA), 16384), g_lo = desc_lo(smem_u32(sG), 16384);
  float acc[32];
  acc_zero(acc);
  for (int i = 0; i < my_tiles; ++i) {
    const int tile = (int)blockIdx.x + i * (int)gridDim.x;
    const int seg = tile % segs, row = tile / segs;
    const int n = row / g.H, y = row - n * g.H;
    if (threadIdx.x == 0) {
      const int q0 = (n * (g.H + 2) + y + 1) * (g.W + 2) + 1 + seg * 128;
      mbar_arrive_expect_tx(g_full, 16384);
      tma_load_2d(sG, &tmG, 0, q0, g_full);
    }
    build_im2col_row(sA, px, I1, I2, n, y, seg * 128 + px, g.H, g.W, true);
    fence_proxy_async();
    __syncthreads();
    mbar_wait(g_full, i & 1);
    acc_fence(acc);
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
      wgmma_bf16<64, 1, 1>(acc, desc_from_lo(a_lo + kk * 128), desc_from_lo(g_lo + kk * 128), 1u);
    wg_commit();
    wg_wait<0>();
    acc_fence(acc);
    __syncthreads();                         // every thread's MMAs are done before the tiles are rebuilt
  }
  {
    // this CTA's slab of the scratch buffer: rows 0..17 = dW[k][co], row 18 = db[co] (CTAs without tiles store zeros); the
    // launcher adds the slabs in CTA order (slab_reduce)
    // the drained tiles hold the transpose block
    float* stg = reinterpret_cast<float*>(base);
    stage_acc64(acc, 0, stg);
    __syncthreads();
    const int r = 32 * (warp & 1) + lane, c = warp >> 1;
    float v[32];
    stg_read32(stg, r, c * 32, v);
    if (r <= 18) {
      float4* dst = reinterpret_cast<float4*>(slab + (size_t)blockIdx.x * kConv1SlabFloats + r * 64 + c * 32);
#pragma unroll
      for (int j = 0; j < 8; ++j) dst[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
    }
  }
}

}  // namespace tc
}  // namespace udh
