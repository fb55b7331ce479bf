// Error-compensated wgmma weight-gradient kernels (UDH_NUMERIC_BF16X3) on two-limb padded streams.
//
//   dW[tap][ci][co] = sum_q X[q + off_tap][ci] * G[q][co]   with   X = X_hi + X_lo,  G = G_hi + G_lo
// evaluated as three passes  X_lo.G_hi + X_hi.G_hi + X_hi.G_lo  into the SAME fp32 accumulators, which stay in registers
// for the CTA's whole run (split-K over CTAs, one group per CTA, partial sums summed in CTA order) — see
// wgrad_tc_kernels.cuh for the operand formulation (MN-major operands, one tap or the ones block per warpgroup, N = 192
// for the 64 -> 64 layers).
//
// Shared memory holds ONE buffer per (operand, limb) — X_hi, X_lo, G_hi, G_lo — each with its own full/empty mbarrier
// pair.  The pass order (X_lo,G_hi) -> (X_hi,G_hi) -> (X_hi,G_lo) staggers their lifetimes: X_lo is free after the first
// third of an item, G_hi after the second, X_hi / G_lo at its end, and each is needed again one third later than it was
// released at the earliest, so every refill runs under the MMAs of another pass although nothing is double-buffered.
//
// Bias gradient: db = sum_q G[q] = ones.(G_hi + G_lo).  The constant-one rows ride along as an extra M block of the X_hi
// passes; in the X_lo pass that M block reads a block of zeros.  Both constant blocks are 16 rows (one k-step) long: every
// k-step reads the same 2 KB.
#pragma once
#include "wgrad_tc_kernels.cuh"

namespace udh {
namespace tc {

constexpr int kConstBlockBytes = 2048;     // 16 positions x 64 channels x 2 bytes

__device__ __forceinline__ void fill_const_blocks(uint8_t* sOnes, uint8_t* sZeros, uint32_t one_pair) {
  uint32_t* o = reinterpret_cast<uint32_t*>(sOnes);
  uint32_t* z = reinterpret_cast<uint32_t*>(sZeros);
  for (int i = threadIdx.x; i < kConstBlockBytes / 4; i += blockDim.x) { o[i] = one_pair; z[i] = 0u; }
  fence_proxy_async();                                          // generic-proxy writes -> visible to the tensor (async) proxy
}
template <int FMT> __host__ __device__ constexpr uint32_t one_pair_bits() { return FMT == kFmtBF16 ? 0x3F803F80u : 0x3C003C00u; }

// buffer indices
constexpr int kXH = 0, kXL = 1, kGH = 2, kGL = 3;

// ---------------------------------------------------------------------------------------------------------------------
// generic kernel: N_OUT = 128; CBX = 1 (64 -> 128: two taps per group) or 2 (128 -> 128: one tap per group + ones group)
template <int N_OUT, int CBX, int T, int FMT_X, int FMT_G>
__global__ void __launch_bounds__(384, 1)
tc_wgrad_x3_kernel(const __grid_constant__ CUtensorMap tmX128, const __grid_constant__ CUtensorMap tmXhh,
                   const __grid_constant__ CUtensorMap tmG, const WgradGeom g, float* __restrict__ slab) {
  static_assert(FMT_X == kFmtBF16 && FMT_G == kFmtBF16, "wgmma multiplies limbs of one format");
  constexpr int CBO = N_OUT / 64;
  extern __shared__ uint8_t raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~(uintptr_t)1023);
  const int xblk_bytes = g.xrows * 128;                         // one 64-channel block of one limb of X
  constexpr int gblk_bytes = T * 128 * 128;                     // one 64-channel block of one limb of G
  const int xl_bytes = CBX * xblk_bytes, gl_bytes = CBO * gblk_bytes;
  uint8_t* sX[2] = {base, base + xl_bytes};                     // [limb][CBX blocks]
  uint8_t* sG[2] = {base + 2 * (size_t)xl_bytes, base + 2 * (size_t)xl_bytes + gl_bytes};
  uint8_t* sOnes = sG[1] + gl_bytes;
  uint8_t* sZeros = sOnes + kConstBlockBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sZeros + kConstBlockBytes);
  uint64_t* full = bars;        // [4]
  uint64_t* empty = bars + 4;   // [4]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int sl = 0;
  while (sl + 1 < g.num_slices && (int)blockIdx.x >= g.slice_cta[sl + 1]) ++sl;
  const int bx = (int)blockIdx.x - g.slice_cta[sl], gxs = g.slice_cta[sl + 1] - g.slice_cta[sl];
  const int gi = g.slice_group[sl];                             // this CTA's group

  fill_const_blocks(sOnes, sZeros, one_pair_bits<FMT_X>());
  if (threadIdx.x == 0) {
    for (int i = 0; i < 4; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 256); }
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) { prefetch_tmap(&tmX128); prefetch_tmap(&tmXhh); prefetch_tmap(&tmG); }
  __syncthreads();
  pdl_wait();                  // predecessor grid complete: global memory may be touched from here on
  pdl_trigger();
  const int my_items = (g.num_items - bx + gxs - 1) / gxs;

  if (warp < 4) {
    regs_dec<40>();
    if (warp == 0 && lane == 0) {
      auto load_x = [&](int l, int q0, uint32_t par) {
        mbar_wait(&empty[l], par);
        mbar_arrive_expect_tx(&full[l], (uint32_t)xl_bytes);
        for (int cb = 0; cb < CBX; ++cb) {
          uint8_t* dst = sX[l] + (size_t)cb * xblk_bytes;
          const int c0 = (l * CBX + cb) * 64;
          tma_load_2d(dst, &tmXhh, c0, q0 - g.hh, &full[l]);
          for (int t = 0; t < T; ++t) tma_load_2d(dst + (size_t)(g.hh + t * 128) * 128, &tmX128, c0, q0 + t * 128, &full[l]);
          tma_load_2d(dst + (size_t)(g.hh + T * 128) * 128, &tmXhh, c0, q0 + T * 128, &full[l]);
        }
      };
      auto load_g = [&](int l, int q0, uint32_t par) {
        mbar_wait(&empty[2 + l], par);
        mbar_arrive_expect_tx(&full[2 + l], (uint32_t)gl_bytes);
        for (int cb = 0; cb < CBO; ++cb)
          for (int t = 0; t < T; ++t)
            tma_load_2d(sG[l] + (size_t)cb * gblk_bytes + (size_t)t * 16384, &tmG, (l * CBO + cb) * 64, q0 + t * 128, &full[2 + l]);
      };
      for (int it = 0; it < my_items; ++it) {
        const int q0 = (bx + it * gxs) * T * 128;
        const uint32_t par = (it & 1) ^ 1;
        load_x(1, q0, par);      // in the order the MMA passes release the buffers
        load_g(0, q0, par);
        load_x(0, q0, par);
        load_g(1, q0, par);
      }
    }
  } else {                                                      // (CTAs without items store zero slabs)
    regs_inc<232>();
    const int cw = (warp - 4) >> 2;
    // A operand of this warpgroup: a row shift of X (channel block xcb), the constant block (ones in the X_hi passes, zeros
    // in the X_lo pass: the constant-one channel has no lo limb), or — for the M = 64 ones group — the ones block, which
    // only the X_hi passes multiply
    int off = 0, xcb = 0, mode = 0;                             // mode 0: X rows; 1: constant block; 2: ones group
    if (CBX == 1) {
      const int tap = 2 * gi + cw;
      if (tap == 9) mode = 1;
      else off = (tap / 3 - 1) * g.Wp + (tap % 3 - 1);
    } else if (gi < 9) {
      off = (gi / 3 - 1) * g.Wp + (gi % 3 - 1);
      xcb = cw;
    } else {
      mode = 2;
    }
    const uint32_t ones_addr = smem_u32(sOnes), zeros_addr = smem_u32(sZeros);
    float acc[N_OUT / 2];
    acc_zero(acc);
    for (int it = 0; it < my_items; ++it) {
      const uint32_t par = it & 1;
#pragma unroll 1
      for (int pass = 0; pass < 3; ++pass) {
        const int xl = pass == 0 ? 1 : 0;                       // X limb of this pass
        const int gl_ = pass == 2 ? 1 : 0;                      // G limb of this pass
        if (pass == 0) { mbar_wait(&full[kXL], par); mbar_wait(&full[kGH], par); }
        else if (pass == 1) mbar_wait(&full[kXH], par);
        else mbar_wait(&full[kGL], par);
        if (!(mode == 2 && xl)) {
          const uint32_t x_addr = smem_u32(sX[xl]);
          const uint32_t g_addr = smem_u32(sG[gl_]);
          const uint32_t const_addr = xl ? zeros_addr : ones_addr;
          acc_fence(acc);
          wg_fence();
#pragma unroll 1
          for (int t = 0; t < T; ++t) {
            const uint32_t b_lo = desc_lo(g_addr + (uint32_t)t * 16384, (uint32_t)gblk_bytes);
            const uint32_t a_start = x_addr + (uint32_t)xcb * xblk_bytes + (uint32_t)(g.hh + t * 128 + off) * 128;
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {                     // 16 positions = 2048 bytes per k-step
              const uint32_t a_lo = mode == 0 ? desc_lo(a_start + kk * 2048, 0)
                                  : desc_lo(mode == 1 ? const_addr : ones_addr, 0);
              wgmma_bf16<N_OUT, 1, 1>(acc, desc_from_lo(a_lo), desc_from_lo(b_lo + kk * 128), 1u);
            }
          }
          wg_commit();
          wg_wait<0>();
          acc_fence(acc);
        }
        if (pass == 0) mbar_arrive(&empty[kXL]);
        else if (pass == 1) mbar_arrive(&empty[kGH]);
        else { mbar_arrive(&empty[kXH]); mbar_arrive(&empty[kGL]); }
      }
    }
    float* mine = slab + (size_t)blockIdx.x * 128 * N_OUT + (size_t)cw * 64 * N_OUT;
    store_acc(acc, [&](int r, int c) -> float* { return mine + (size_t)r * N_OUT + c; });
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// 64 -> 64 channel layers: the N = 192 formulation of tc_wgrad64_kernel (B = three row shifts of G; group 0 = [X[q - Wp] |
// X[q]], group 1 = [X[q + Wp] | constant block]; even CTAs own group 0, odd CTAs group 1), with the limb passes above.
template <int T, int FMT_X, int FMT_G>
__global__ void __launch_bounds__(384, 1)
tc_wgrad64_x3_kernel(const __grid_constant__ CUtensorMap tmX128, const __grid_constant__ CUtensorMap tmXhh,
                     const __grid_constant__ CUtensorMap tmG136, const Wgrad64Geom g, float* __restrict__ slab) {
  static_assert(T == 2, "G is staged as two 136-row boxes");
  static_assert(FMT_X == kFmtBF16 && FMT_G == kFmtBF16, "wgmma multiplies limbs of one format");
  extern __shared__ uint8_t raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~(uintptr_t)1023);
  const int xblk_bytes = g.xrows * 128;
  constexpr int kGRows = T * 128 + 16;                          // 8 halo rows on each side
  constexpr int gblk_bytes = kGRows * 128;
  uint8_t* sX[2] = {base, base + xblk_bytes};
  uint8_t* sG[2] = {base + 2 * (size_t)xblk_bytes, base + 2 * (size_t)xblk_bytes + gblk_bytes};
  uint8_t* sOnes = sG[1] + gblk_bytes;
  uint8_t* sZeros = sOnes + kConstBlockBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sZeros + kConstBlockBytes);
  uint64_t* full = bars;        // [4]
  uint64_t* empty = bars + 4;   // [4]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gl = (int)blockIdx.x & 1, bx = (int)blockIdx.x >> 1, gxs = (int)gridDim.x >> 1;

  fill_const_blocks(sOnes, sZeros, one_pair_bits<FMT_X>());
  if (threadIdx.x == 0) {
    for (int i = 0; i < 4; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 256); }
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) { prefetch_tmap(&tmX128); prefetch_tmap(&tmXhh); prefetch_tmap(&tmG136); }
  __syncthreads();
  pdl_wait();                  // predecessor grid complete: global memory may be touched from here on
  pdl_trigger();
  const int my_items = (g.num_items - bx + gxs - 1) / gxs;

  if (warp < 4) {
    regs_dec<40>();
    if (warp == 0 && lane == 0) {
      auto load_x = [&](int l, int q0, uint32_t par) {
        mbar_wait(&empty[l], par);
        mbar_arrive_expect_tx(&full[l], (uint32_t)xblk_bytes);
        uint8_t* dst = sX[l];
        tma_load_2d(dst, &tmXhh, l * 64, q0 - g.hh, &full[l]);
        for (int t = 0; t < T; ++t) tma_load_2d(dst + (size_t)(g.hh + t * 128) * 128, &tmX128, l * 64, q0 + t * 128, &full[l]);
        tma_load_2d(dst + (size_t)(g.hh + T * 128) * 128, &tmXhh, l * 64, q0 + T * 128, &full[l]);
      };
      auto load_g = [&](int l, int q0, uint32_t par) {
        mbar_wait(&empty[2 + l], par);
        mbar_arrive_expect_tx(&full[2 + l], (uint32_t)gblk_bytes);
        tma_load_2d(sG[l], &tmG136, l * 64, q0 - 8, &full[2 + l]);
        tma_load_2d(sG[l] + 136 * 128, &tmG136, l * 64, q0 + 128, &full[2 + l]);
      };
      for (int it = 0; it < my_items; ++it) {
        const int q0 = (bx + it * gxs) * T * 128;
        const uint32_t par = (it & 1) ^ 1;
        load_x(1, q0, par);
        load_g(0, q0, par);
        load_x(0, q0, par);
        load_g(1, q0, par);
      }
    }
  } else {                                                      // (CTAs without items store zero slabs)
    regs_inc<232>();
    const int cw = (warp - 4) >> 2;
    const int shift = gl == 0 ? (cw == 0 ? -g.Wp : 0) : g.Wp;
    const bool cst = gl == 1 && cw == 1;                        // constant block (ones / zeros) instead of X rows
    const uint32_t ones_addr = smem_u32(sOnes), zeros_addr = smem_u32(sZeros);
    float acc[96];
    acc_zero(acc);
    for (int it = 0; it < my_items; ++it) {
      const uint32_t par = it & 1;
#pragma unroll 1
      for (int pass = 0; pass < 3; ++pass) {
        const int xl = pass == 0 ? 1 : 0;
        const int gl_ = pass == 2 ? 1 : 0;
        if (pass == 0) { mbar_wait(&full[kXL], par); mbar_wait(&full[kGH], par); }
        else if (pass == 1) mbar_wait(&full[kXH], par);
        else mbar_wait(&full[kGL], par);
        const uint32_t x_addr = smem_u32(sX[xl]);
        const uint32_t g_addr = smem_u32(sG[gl_]);
        const uint32_t const_addr = xl ? zeros_addr : ones_addr;
        acc_fence(acc);
        wg_fence();
        // unrolled: a loop back-edge between the MMAs would make ptxas wait for them (C7519)
#pragma unroll
        for (int t = 0; t < T; ++t) {
          const uint32_t b_lo = desc_lo(g_addr + (uint32_t)(8 + t * 128 - 1) * 128, 128);     // G[q-1] | G[q] | G[q+1]
          const uint32_t a_start = x_addr + (uint32_t)(g.hh + t * 128 + shift) * 128;
#pragma unroll
          for (int kk = 0; kk < 8; ++kk) {
            const uint32_t a_lo = desc_lo(cst ? const_addr : a_start + kk * 2048, 0);
            wgmma_bf16<192, 1, 1>(acc, desc_from_lo(a_lo), desc_from_lo(b_lo + kk * 128), 1u);
          }
        }
        wg_commit();
        wg_wait<0>();
        acc_fence(acc);
        if (pass == 0) mbar_arrive(&empty[kXL]);
        else if (pass == 1) mbar_arrive(&empty[kGH]);
        else { mbar_arrive(&empty[kXH]); mbar_arrive(&empty[kGL]); }
      }
    }
    float* mine = slab + (size_t)blockIdx.x * kWgrad64SlabFloats;
    store_acc(acc, [&](int r, int c) -> float* {
      const int m = 64 * cw + r, ci = m & 63, jb = c >> 6, co = c & 63;   // N block jb: G shift jb - 1 -> kx = 1 - jb
      if (gl == 1 && m >= 64) return (m == 64 && jb == 1) ? mine + 3 * 4096 + co : nullptr;   // ones rows: db
      const int ky = gl == 0 ? (m >> 6) - 1 : 1;
      const int tap = (ky + 1) * 3 + (2 - jb);
      return mine + ((size_t)(tap - 6 * gl) * 64 + ci) * 64 + co;
    });
  }
}

}  // namespace tc
}  // namespace udh
