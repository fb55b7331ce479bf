// wgmma weight-gradient kernel on the padded bf16 streams (see conv_tc_kernels.cuh for the layout).
//
//   dW[tap][ci][co] = sum_q X[q + off_tap][ci] * G[q][co],   off_tap = (ky-1)*Wp + (kx-1)
// summed over EVERY flattened position q: G is zero on the borders, so border terms vanish and no masking is needed.
// Positions are the contraction (K) dimension, channels are contiguous in memory, so both operands are MN-major:
//   A = rows of X shifted by off_tap (M = input channels), B = rows of G (N = output channels), K = 16 positions / MMA.
// A GROUP is 128 accumulator rows; MMA warpgroup cw owns rows [64 cw, 64 cw + 64):
//   Cin = 64  : TWO TAPS per group — warpgroup 1 reads the same staged X rows shifted by (off_b - off_a); the odd tap 8 is
//               paired with a block of ones, whose 64 identical result rows are the bias gradient sum_q G[q][co];
//   Cin = 128 : one tap per group, the two 64-channel blocks of X are the two warpgroups' A operands; a tenth group
//               multiplies the ones block with G (bias gradient, its first row is used).
// Every CTA owns ONE group (the accumulators of a group fill the MMA warpgroups' registers): the groups are slices of the
// 1-D grid, each with a share of the CTAs, and every CTA reduces its group over its positions (split-K) into its own slab of
// a scratch buffer; the launcher adds the slabs to the fp32 gradient buffer in CTA order.
// warpgroup 0: TMA producer (warp 0) | warpgroups 1-2: MMA + epilogue.
#pragma once
#include "tc_common.cuh"

namespace udh {
namespace tc {

struct WgradGeom {
  int Wp, Q, hh;
  int num_items;     // ceil(ceil(Q/128) / T)
  int xrows;         // T*128 + 2*hh rows staged per 64-channel block of X
  int num_groups;    // CBX == 1: 5 (4 tap pairs + tap 8 | ones);  CBX == 2: 10 (9 taps + ones)
  // slice s owns groups [slice_group[s], slice_group[s+1]) and CTAs [slice_cta[s], slice_cta[s+1]) of the 1-D grid
  // (CTA counts proportional to the slice's group count, so every CTA issues about the same number of MMAs); the kernels
  // take one group per slice.
  int num_slices;
  int slice_group[11];
  int slice_cta[11];
};

// Every CTA stores its group's accumulators in its own slab of a scratch buffer; the launcher then adds the slabs to the
// fp32 gradient buffer in a fixed order (slab_reduce), so the gradient does not depend on CTA timing.
//   generic kernels: slab = the group's 128 rows x N_OUT columns, in the order of the gradient rows they feed;
//   N = 192 kernels: slab = the group's taps in the HWIO layout of dW (group 0: taps 0-5; group 1: taps 6-8, then db).
constexpr int kWgrad64SlabFloats = 6 * 64 * 64;

template <int N_OUT, int CBX, int T>
__global__ void __launch_bounds__(384, 1)
tc_wgrad_kernel(const __grid_constant__ CUtensorMap tmX128, const __grid_constant__ CUtensorMap tmXhh,
                const __grid_constant__ CUtensorMap tmG, const WgradGeom g, float* __restrict__ slab) {
  constexpr int CBO = N_OUT / 64;
  extern __shared__ uint8_t raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~(uintptr_t)1023);
  const int xblk_bytes = g.xrows * 128;                         // one 64-channel block of X of one stage
  const int gblk_bytes = T * 128 * 128;                         // one 64-channel block of G of one stage
  const int stage_bytes = CBX * xblk_bytes + CBO * gblk_bytes;
  uint8_t* sStage = base;                                       // [2][ X: CBX blocks | G: CBO blocks ]
  uint8_t* sOnes = base + 2 * (size_t)stage_bytes;              // [128][64] bf16 ones
  uint64_t* bars = reinterpret_cast<uint64_t*>(sOnes + 16384);
  uint64_t* full = bars;        // [2]
  uint64_t* empty = bars + 2;   // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int sl = 0;
  while (sl + 1 < g.num_slices && (int)blockIdx.x >= g.slice_cta[sl + 1]) ++sl;
  const int bx = (int)blockIdx.x - g.slice_cta[sl], gxs = g.slice_cta[sl + 1] - g.slice_cta[sl];
  const int gi = g.slice_group[sl];                             // this CTA's group

  {
    // ones block: every 16-byte chunk is identical, so the 128-byte swizzle leaves it unchanged
    uint32_t* o = reinterpret_cast<uint32_t*>(sOnes);
    for (int i = threadIdx.x; i < 16384 / 4; i += blockDim.x) o[i] = 0x3F803F80u;
    fence_proxy_async();                                        // generic-proxy writes -> visible to the tensor (async) proxy
  }
  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 256); }
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
      for (int it = 0; it < my_items; ++it) {
        const int s = it & 1;
        const int q0 = (bx + it * gxs) * T * 128;
        mbar_wait(&empty[s], ((it >> 1) & 1) ^ 1);
        mbar_arrive_expect_tx(&full[s], (uint32_t)stage_bytes);
        uint8_t* st = sStage + (size_t)s * stage_bytes;
        for (int cb = 0; cb < CBX; ++cb) {
          uint8_t* dst = st + (size_t)cb * xblk_bytes;
          tma_load_2d(dst, &tmXhh, cb * 64, q0 - g.hh, &full[s]);
          for (int t = 0; t < T; ++t) tma_load_2d(dst + (size_t)(g.hh + t * 128) * 128, &tmX128, cb * 64, q0 + t * 128, &full[s]);
          tma_load_2d(dst + (size_t)(g.hh + T * 128) * 128, &tmXhh, cb * 64, q0 + T * 128, &full[s]);
        }
        for (int cb = 0; cb < CBO; ++cb)
          for (int t = 0; t < T; ++t)
            tma_load_2d(st + (size_t)CBX * xblk_bytes + (size_t)cb * gblk_bytes + (size_t)t * 16384, &tmG, cb * 64, q0 + t * 128, &full[s]);
      }
    }
  } else {                                                      // (CTAs without items store zero slabs)
    regs_inc<232>();
    const int cw = (warp - 4) >> 2;
    const uint32_t ones_addr = smem_u32(sOnes);
    // A operand of this warpgroup: a row shift of X (channel block xcb), or the ones block
    int off = 0, xcb = 0;
    bool ones = false;
    if (CBX == 1) {
      const int tap = 2 * gi + cw;
      if (tap == 9) ones = true;
      else off = (tap / 3 - 1) * g.Wp + (tap % 3 - 1);
    } else if (gi < 9) {
      off = (gi / 3 - 1) * g.Wp + (gi % 3 - 1);
      xcb = cw;
    } else {
      ones = true;
    }
    float acc[N_OUT / 2];
    acc_zero(acc);
    for (int it = 0; it < my_items; ++it) {
      const int s = it & 1;
      mbar_wait(&full[s], (it >> 1) & 1);
      const uint32_t x_addr = smem_u32(sStage + (size_t)s * stage_bytes);
      const uint32_t g_addr = x_addr + (uint32_t)(CBX * xblk_bytes);
      acc_fence(acc);
      wg_fence();
#pragma unroll 1
      for (int t = 0; t < T; ++t) {
        const uint32_t a_start = ones ? ones_addr : x_addr + (uint32_t)xcb * xblk_bytes + (uint32_t)(g.hh + t * 128 + off) * 128;
        const uint32_t a_lo = desc_lo(a_start, 0);
        const uint32_t b_lo = desc_lo(g_addr + (uint32_t)t * 16384, (uint32_t)gblk_bytes);
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)                     // 16 positions = 2048 bytes = 128 sixteen-byte units per k-step
          wgmma_bf16<N_OUT, 1, 1>(acc, desc_from_lo(a_lo + kk * 128), desc_from_lo(b_lo + kk * 128), 1u);
      }
      wg_commit();
      wg_wait<0>();
      acc_fence(acc);
      mbar_arrive(&empty[s]);
    }
    float* mine = slab + (size_t)blockIdx.x * 128 * N_OUT + (size_t)cw * 64 * N_OUT;
    store_acc(acc, [&](int r, int c) -> float* { return mine + (size_t)r * N_OUT + c; });
  }
}


// ---------------------------------------------------------------------------------------------------------------------
// 64 -> 64 channel layers (conv1_2, conv2_1, conv2_2): N = 192 variant.
// The N side is widened: B is THREE row shifts of the gradient rows, c = -1, 0, +1 (three 64-wide MN blocks, leading-dimension
// byte offset = one 128-byte row), A is a row shift of X (one per MMA warpgroup: the ky and ky' rows of the 3x3 window).  Since
//   sum_q X[q + a][ci] * G[q + c][co]  =  dW at tap offset (a - c),
// one (M128, N192) group yields the six taps (ky, ky') x (kx = -c), and the whole 3x3 window + bias gradient takes two groups:
//   group 0: A = X[q - Wp] | X[q]          -> taps ky = -1, 0 ; kx = +1, 0, -1 (N blocks 0, 1, 2)
//   group 1: A = X[q + Wp] | ones          -> taps ky = +1    ; rows 64.. = bias gradient (taken from N block 1)
// G needs one halo row on each side (8 are staged to keep the 1024-byte swizzle-atom alignment of the TMA boxes).
struct Wgrad64Geom {
  int Wp, Q, hh;
  int num_items;     // ceil(ceil(Q/128) / T)
  int xrows;         // T*128 + 2*hh
};

template <int T>
__global__ void __launch_bounds__(384, 1)
tc_wgrad64_kernel(const __grid_constant__ CUtensorMap tmX128, const __grid_constant__ CUtensorMap tmXhh,
                  const __grid_constant__ CUtensorMap tmG136, const Wgrad64Geom g, float* __restrict__ slab) {
  static_assert(T == 2, "G is staged as two 136-row boxes");
  extern __shared__ uint8_t raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~(uintptr_t)1023);
  const int xblk_bytes = g.xrows * 128;
  constexpr int kGRows = T * 128 + 16;                          // 8 halo rows on each side
  constexpr int gblk_bytes = kGRows * 128;
  const int stage_bytes = xblk_bytes + gblk_bytes;
  uint8_t* sStage = base;                                       // [2][ X rows | G rows ]
  uint8_t* sOnes = base + 2 * (size_t)stage_bytes;              // [128][64] bf16 ones
  uint64_t* bars = reinterpret_cast<uint64_t*>(sOnes + 16384);
  uint64_t* full = bars;        // [2]
  uint64_t* empty = bars + 2;   // [2]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // even CTAs own group 0, odd CTAs group 1 (a group's 128 x 192 accumulators fill the MMA warpgroups' registers)
  const int gl = (int)blockIdx.x & 1, bx = (int)blockIdx.x >> 1, gxs = (int)gridDim.x >> 1;

  {
    uint32_t* o = reinterpret_cast<uint32_t*>(sOnes);
    for (int i = threadIdx.x; i < 16384 / 4; i += blockDim.x) o[i] = 0x3F803F80u;
    fence_proxy_async();
  }
  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 256); }
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
      for (int it = 0; it < my_items; ++it) {
        const int s = it & 1;
        const int q0 = (bx + it * gxs) * T * 128;
        mbar_wait(&empty[s], ((it >> 1) & 1) ^ 1);
        mbar_arrive_expect_tx(&full[s], (uint32_t)stage_bytes);
        uint8_t* dst = sStage + (size_t)s * stage_bytes;
        tma_load_2d(dst, &tmXhh, 0, q0 - g.hh, &full[s]);
        for (int t = 0; t < T; ++t) tma_load_2d(dst + (size_t)(g.hh + t * 128) * 128, &tmX128, 0, q0 + t * 128, &full[s]);
        tma_load_2d(dst + (size_t)(g.hh + T * 128) * 128, &tmXhh, 0, q0 + T * 128, &full[s]);
        uint8_t* gd = dst + xblk_bytes;
        tma_load_2d(gd, &tmG136, 0, q0 - 8, &full[s]);
        tma_load_2d(gd + 136 * 128, &tmG136, 0, q0 + 128, &full[s]);
      }
    }
  } else {                                                      // (CTAs without items store zero slabs)
    regs_inc<232>();
    const int cw = (warp - 4) >> 2;
    const uint32_t ones_addr = smem_u32(sOnes);
    // rows of the group: group 0 = [X[q - Wp] | X[q]], group 1 = [X[q + Wp] | ones]
    const int shift = gl == 0 ? (cw == 0 ? -g.Wp : 0) : g.Wp;
    const bool ones = gl == 1 && cw == 1;
    float acc[96];
    acc_zero(acc);
    for (int it = 0; it < my_items; ++it) {
      const int s = it & 1;
      mbar_wait(&full[s], (it >> 1) & 1);
      const uint32_t x_addr = smem_u32(sStage + (size_t)s * stage_bytes);
      const uint32_t g_addr = x_addr + (uint32_t)xblk_bytes;
      acc_fence(acc);
      wg_fence();
#pragma unroll 1
      for (int t = 0; t < T; ++t) {
        const uint32_t b_lo = desc_lo(g_addr + (uint32_t)(8 + t * 128 - 1) * 128, 128);     // G[q-1] | G[q] | G[q+1]
        const uint32_t a_lo = desc_lo(ones ? ones_addr : x_addr + (uint32_t)(g.hh + t * 128 + shift) * 128, 0);
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)
          wgmma_bf16<192, 1, 1>(acc, desc_from_lo(a_lo + kk * 128), desc_from_lo(b_lo + kk * 128), 1u);
      }
      wg_commit();
      wg_wait<0>();
      acc_fence(acc);
      mbar_arrive(&empty[s]);
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
