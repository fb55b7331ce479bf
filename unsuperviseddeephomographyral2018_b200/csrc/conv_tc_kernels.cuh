// wgmma implicit-GEMM 3x3 convolution over a flattened, zero-bordered NHWC bf16 activation ("padded stream").
//
// Layout.  An activation [B,H,W,C] is stored as [B][H+2][W+2][C] bf16 with zero borders; flattened, it is a matrix
// X[Q = B*(H+2)*(W+2) positions][C].  With Wp = W+2, the input of tap (ky,kx) for output position q is simply row
// q + (ky-1)*Wp + (kx-1): every tap is a ROW SHIFT of the same matrix, borders supply the zero padding, and images
// never bleed into each other.  Outputs at border positions are computed but not stored (~3 % waste at W = 128).
//
// Kernel.  One persistent CTA per SM walks work items of T consecutive 128-position tiles:
//   * TMA (SWIZZLE_128B) stages rows [q0-hh, q0+128T+hh) of X once per item into a linear smem buffer (per 64-channel
//     block); all 9 taps are wgmma shared-memory descriptors whose START ADDRESS is shifted by whole 128-byte rows
//     inside that buffer (the hardware swizzles on absolute smem address bits, so unaligned row starts need no
//     base_offset).  L2->smem traffic is ~(1 + 2hh/128T)x the activation instead of 9x.
//   * weights [tap][cblock][Cout][64] are either resident in smem (<= 144 KiB) or streamed through a small TMA ring,
//     each streamed k-block being reused by the T tiles of the item (T accumulators per thread);
//   * two MMA warpgroups each own 64 of the 128 rows of every tile; their fp32 accumulators live in registers.  A
//     warpgroup releases the staged rows as soon as its MMAs are complete, so the TMA thread loads the next item's rows
//     while the epilogue (same warpgroups) drains the accumulators through a small transpose block (stage_acc64).
//   warpgroup 0: TMA producer (warp 0) | warpgroups 1-2: MMA + epilogue.
//
// Row-tile variants (W == 128, T == 2, 64 -> 64 channels: conv1_2).  ROWS = 1: forward fused with pool1; ROWS = 2: dgrad
// with the plain bias / mask / TMA-store epilogue.  An item is the interior of two consecutive image rows (2y, 2y+1):
// tile t starts at the first interior position of row 2y+t, i.e. the two tiles are Wp (not 128) rows apart in the same
// staged buffer, no border position is computed, and the epilogue thread of column x holds both rows of that column.
//   * ROWS = 1 epilogue: bias + ReLU, 2x2 maximum (vertical in registers, horizontal with one lane exchange), then the
//     POOLED padded stream plus the 3-bit routing codes of the max-pool backward are written — the full-resolution
//     activation is never written or re-read.
//   * MMA schedule: a vertical tap is exactly one tile here, so the MMAs are organised by INPUT row instead of output
//     row.  Input row r feeds output rows r-1, r, r+1 through the ky = +1, 0, -1 weights; for one kx the input rows
//     2y-1 .. 2y+2 issue (N64 | N128 | N128 | N64) MMAs whose N = 128 operands are two adjacent weight blocks writing the
//     two adjacent accumulators at once: 4 MMAs per k-step and kx instead of 6.  Weights are packed in
//     (kx, ky descending) block order (pack_weights_kernel, rowtile = 1).
#pragma once
#include "tc_common.cuh"

namespace udh {
namespace tc {

struct ConvGeom {
  int B, H, W, Hp, Wp;     // Hp = H+2, Wp = W+2
  int Q;                   // B*Hp*Wp flattened positions
  int hh;                  // halo rows staged on each side: round_up(Wp+1, 8)
  int num_items;           // ceil(ceil(Q/128) / T)
  int abuf_rows;           // T*128 + 2*hh
};

constexpr int kNumWStages = 3;

constexpr int kEpiStageBytes = 4 * 32 * 128;   // TMA-store staging: 32 rows x 128 B per epilogue warp

template <int N_OUT, int CB, int T, bool WRES>
struct ConvSmem {
  static constexpr int kWBytesPerKb = N_OUT * 128;
  static constexpr int kWBytes = WRES ? 9 * CB * kWBytesPerKb : kNumWStages * kWBytesPerKb;
  static size_t bytes(int abuf_rows, bool tma_epi) {
    return 1024 + (size_t)CB * abuf_rows * 128 + kWBytes + (tma_epi ? kEpiStageBytes : 0) + 2 * kStgBytes + 256;
  }
};

// TMA_EPI: the epilogue stages each warp's 32 x 64-channel bf16 block in (swizzled) shared memory and writes it with one
// TMA store (full 128-byte lines, asynchronous); the ReLU-mask block of a dgrad is fetched the same way round (coalesced
// 512-byte warp loads into the staging block).  Without it each lane stores its own 64 bytes at a 128-byte stride.
// threads per CTA: the producer warpgroup + two MMA / epilogue warpgroups.  In the epilogue warp w of MMA warpgroup cw
// handles row quarter ew = 2 cw + (w & 1) of the tile and every second 32-column chunk (eg = w >> 1) of the accumulator.
template <bool TMA_EPI> __host__ __device__ constexpr int conv_threads() { return 384; }

template <int N_OUT, int CB, int T, bool WRES, bool TMA_EPI, int ROWS = 0>
__global__ void __launch_bounds__(conv_threads<TMA_EPI>(), 1)
tc_conv_kernel(const __grid_constant__ CUtensorMap tmA128, const __grid_constant__ CUtensorMap tmAhh,
               const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmOut, const ConvGeom g,
               const float* __restrict__ bias, const __nv_bfloat16* __restrict__ mask_src, const uint32_t* __restrict__ mask_bits,
               uint32_t* __restrict__ mask_out, __nv_bfloat16* __restrict__ out_bf, float* __restrict__ out_f32, int relu) {
  constexpr bool POOL = ROWS == 1;
  static_assert(ROWS == 0 || (N_OUT == 64 && T == 2 && CB == 1 && WRES), "row tiles: 64 -> 64 channels, two row tiles, resident weights");
  constexpr int kAccRegs = T * N_OUT / 2;                           // fragment of T tiles x 64 rows x N_OUT columns
  extern __shared__ uint8_t raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~(uintptr_t)1023);
  const int abuf_bytes = g.abuf_rows * 128;                       // one 64-channel block
  uint8_t* sA = base;                                             // [CB][abuf_rows][128]
  uint8_t* sW = base + (size_t)CB * abuf_bytes;                   // resident: [9*CB][N_OUT][128]; streamed: [stages][N_OUT][128]
  uint8_t* sEpi = sW + ConvSmem<N_OUT, CB, T, WRES>::kWBytes;      // [4 quarters][32 rows][128 B] (TMA_EPI only)
  float* sStg = reinterpret_cast<float*>(sEpi + (TMA_EPI ? kEpiStageBytes : 0));   // [2 warpgroups][kStgBytes]
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sStg) + 2 * kStgBytes);
  uint64_t* a_full = bars;
  uint64_t* a_empty = bars + 1;
  uint64_t* w_full = bars + 2;        // [kNumWStages] (or [1] resident)
  uint64_t* w_empty = bars + 2 + kNumWStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    mbar_init(a_full, 1); mbar_init(a_empty, 256);
    for (int i = 0; i < kNumWStages; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], 256); }
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) { prefetch_tmap(&tmA128); prefetch_tmap(&tmAhh); prefetch_tmap(&tmW); if (TMA_EPI) prefetch_tmap(&tmOut); }
  __syncthreads();
  const int my_items = (g.num_items - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // items blockIdx.x + i*gridDim.x
  pdl_wait();                  // predecessor grid complete: global memory may be touched from here on
  pdl_trigger();

  if (warp < 4) {
    regs_dec<40>();
    // ===================================== TMA producer =====================================
    if (warp == 0 && lane == 0) {
      if (WRES) {
        mbar_arrive_expect_tx(&w_full[0], 9 * CB * ConvSmem<N_OUT, CB, T, WRES>::kWBytesPerKb);
        for (int kb = 0; kb < 9 * CB; ++kb)
          tma_load_2d(sW + (size_t)kb * N_OUT * 128, &tmW, 0, kb * N_OUT, &w_full[0]);
      }
      uint32_t wcount = 0;
      for (int it = 0; it < my_items; ++it) {
        const int item = (int)blockIdx.x + it * (int)gridDim.x;
        const int q0 = ROWS ? ((item / (g.H >> 1)) * g.Hp + 2 * (item % (g.H >> 1)) + 1) * g.Wp + 1 : item * T * 128;
        mbar_wait(a_empty, (it & 1) ^ 1);
        mbar_arrive_expect_tx(a_full, (uint32_t)(CB * abuf_bytes));
        for (int cb = 0; cb < CB; ++cb) {
          uint8_t* dst = sA + (size_t)cb * abuf_bytes;
          tma_load_2d(dst, &tmAhh, cb * 64, q0 - g.hh, a_full);
          for (int t = 0; t < T; ++t)
            tma_load_2d(dst + (size_t)(g.hh + t * 128) * 128, &tmA128, cb * 64, q0 + t * 128, a_full);
          tma_load_2d(dst + (size_t)(g.hh + T * 128) * 128, &tmAhh, cb * 64, q0 + T * 128, a_full);
        }
        if (!WRES) {
          for (int kb = 0; kb < 9 * CB; ++kb, ++wcount) {
            const int s = wcount % kNumWStages;
            mbar_wait(&w_empty[s], ((wcount / kNumWStages) & 1) ^ 1);
            mbar_arrive_expect_tx(&w_full[s], N_OUT * 128);
            tma_load_2d(sW + (size_t)s * N_OUT * 128, &tmW, 0, kb * N_OUT, &w_full[s]);
          }
        }
      }
    }
  } else {
    regs_inc<232>();
    const int cw = (warp - 4) >> 2;               // MMA warpgroup: rows [64 cw, 64 cw + 64) of every tile
    const int wi = warp & 3;
    const int ew = 2 * cw + (wi & 1);             // row quarter of the tile this warp drains
    const int eg = wi >> 1;                       // 32-column chunk parity this warp drains
    const int erow = 32 * (wi & 1) + lane;        // row of the warpgroup's fragment
    float* stg = sStg + cw * (kStgBytes / 4);
    auto wg_sync = [&]() { named_sync(5 + cw, 128); };
    // ===================================== MMA =====================================
    const uint32_t a_addr0 = smem_u32(sA) + (uint32_t)cw * 64 * 128, w_addr0 = smem_u32(sW);
    if (WRES) mbar_wait(&w_full[0], 0);
    uint32_t wcount = 0;
    float acc[kAccRegs];
    // ===================================== epilogue state =====================================
    const int HpWp = g.Hp * g.Wp;
    uint8_t* estg = sEpi + ew * 4096;             // the quarter's 32 x 128 B TMA-store staging block (1024-byte aligned)
    const uint32_t my_row = smem_u32(estg) + lane * 128;
    const int sw = lane & 7;                      // 128-byte swizzle phase of this lane's row
    const bool issuer = eg == 0 && lane == 0;     // the thread that owns the quarter's TMA-store bulk groups
    auto pair_sync = [&]() { named_sync(1 + ew, 64); };
    bool store_pending = false;
    for (int it = 0; it < my_items; ++it) {
      const int item = (int)blockIdx.x + it * (int)gridDim.x;
      // ReLU-backward mask of a dgrad as 1 bit / element: requested before the MMAs so the load latency hides behind them
      uint32_t mbt[2][N_OUT / 32];
      if (TMA_EPI && !POOL) {
        const int q0w0 = ROWS ? ((item / (g.H >> 1)) * g.Hp + 2 * (item % (g.H >> 1)) + 1) * g.Wp + 1 + ew * 32 : item * T * 128 + ew * 32;
        const int qstep = ROWS ? g.Wp : 128;
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          const int qt = q0w0 + t * qstep + lane;
          const bool ok = mask_bits && t < T && qt < g.Q;
          if (N_OUT == 64) {
            const uint2 m = ok ? __ldg(reinterpret_cast<const uint2*>(mask_bits + (size_t)qt * 2)) : make_uint2(0u, 0u);
            mbt[t][0] = m.x; mbt[t][1] = m.y;
          } else {
            const uint4 m = ok ? __ldg(reinterpret_cast<const uint4*>(mask_bits + (size_t)qt * 4)) : make_uint4(0u, 0u, 0u, 0u);
            mbt[t][0] = m.x; mbt[t][1] = m.y; mbt[t][N_OUT / 32 - 2] = m.z; mbt[t][N_OUT / 32 - 1] = m.w;
          }
        }
      }
      mbar_wait(a_full, it & 1);
      acc_fence(acc);
      if constexpr (ROWS != 0) {
        // acc = [O(2y) | O(2y+1)], 64 columns each
        const uint32_t a_row0 = a_addr0 + (uint32_t)g.hh * 128;                             // first interior position of row 2y
#pragma unroll 1
        for (int kx = 0; kx < 3; ++kx) {
          const uint32_t wk = w_addr0 + (uint32_t)(kx * 3) * 64 * 128;      // blocks ky = +1, 0, -1 of this kx
          //   r =  0: [W(0) | W(-1)] -> O0, O1     r = 1: [W(+1) | W(0)] -> O0, O1     r = -1: W(-1) -> O0     r = 2: W(+1) -> O1
          const uint32_t a0 = desc_lo(a_row0 + (uint32_t)((kx - 1) * 128), 16);
          const uint32_t a1 = desc_lo(a_row0 + (uint32_t)((g.Wp + kx - 1) * 128), 16);
          const uint32_t am = desc_lo(a_row0 + (uint32_t)((-g.Wp + kx - 1) * 128), 16);
          const uint32_t a2 = desc_lo(a_row0 + (uint32_t)((2 * g.Wp + kx - 1) * 128), 16);
          const uint32_t w_p1 = desc_lo(wk, 16), w_0 = desc_lo(wk + 64 * 128, 16), w_m1 = desc_lo(wk + 2 * 64 * 128, 16);
          wg_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_bf16<128, 0, 0>(acc, desc_from_lo(a0 + k * 2), desc_from_lo(w_0 + k * 2), (kx > 0 || k > 0) ? 1u : 0u);
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_bf16<128, 0, 0>(acc, desc_from_lo(a1 + k * 2), desc_from_lo(w_p1 + k * 2), 1u);
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_bf16_head<64, 0, 0>(acc, desc_from_lo(am + k * 2), desc_from_lo(w_m1 + k * 2), 1u);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            Wgmma<64>::run<0, 0>(*reinterpret_cast<float(*)[32]>(&acc[32]), desc_from_lo(a2 + k * 2), desc_from_lo(w_p1 + k * 2), 1u);
          wg_commit();
        }
        wg_wait<0>();
      } else {
        int prev = -1;
        for (int kb = 0; kb < 9 * CB; ++kb) {
          const int tap = kb / CB, cb = kb - tap * CB;
          const int ky = tap / 3, kx = tap - ky * 3;
          const int off = (ky - 1) * g.Wp + (kx - 1);
          uint32_t w_addr;
          int s = 0;
          if (WRES) {
            w_addr = w_addr0 + (uint32_t)kb * N_OUT * 128;
          } else {
            s = wcount % kNumWStages;
            mbar_wait(&w_full[s], (wcount / kNumWStages) & 1);
            w_addr = w_addr0 + (uint32_t)s * N_OUT * 128;
          }
          const uint32_t a_lo = desc_lo(a_addr0 + (uint32_t)cb * abuf_bytes + (uint32_t)(g.hh + off) * 128, 16);
          const uint32_t w_lo = desc_lo(w_addr, 16);
          wg_fence();
#pragma unroll
          for (int t = 0; t < T; ++t) {
#pragma unroll
            for (int k = 0; k < 4; ++k)     // +1024 sixteen-byte units per tile, +2 per 32-byte k-step
              Wgmma<N_OUT>::template run<0, 0>(*reinterpret_cast<float(*)[N_OUT / 2]>(&acc[t * (N_OUT / 2)]),
                                               desc_from_lo(a_lo + t * 1024 + k * 2), desc_from_lo(w_lo + k * 2), (kb > 0 || k > 0) ? 1u : 0u);
          }
          wg_commit();
          if (!WRES) {
            wg_wait<1>();                          // the MMAs of the previous k-block are done: its ring slot is free
            if (prev >= 0) mbar_arrive(&w_empty[prev]);
            prev = s;
            ++wcount;
          }
        }
        wg_wait<0>();
        if (!WRES && prev >= 0) mbar_arrive(&w_empty[prev]);
      }
      acc_fence(acc);
      mbar_arrive(a_empty);                       // staged rows no longer read -> producer loads the next item
      // ===================================== epilogue =====================================
      if constexpr (POOL) {
        const int OH = g.H >> 1, OW = g.W >> 1;
        const int x = ew * 32 + lane;                 // column of this thread (W == 128 == tile rows)
        const int px = x >> 1, odd = x & 1;
        const int n = item / OH, yy = item - n * OH;
        __nv_bfloat16* prow = out_bf + (((size_t)n * (OH + 2) + yy + 1) * (OW + 2) + px + 1) * 64;
        uint32_t* crow = mask_out + (((size_t)n * OH + yy) * OW + px) * 8;
        const int c = eg;
        float v0[32], v1[32];
        wg_sync(); stage_acc64(acc, 0, stg); wg_sync();
        stg_read32(stg, erow, c * 32, v0);
        wg_sync(); stage_acc64(acc, 1, stg); wg_sync();
        stg_read32(stg, erow, c * 32, v1);
        uint32_t code[4] = {0u, 0u, 0u, 0u};
        float m[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const float bj = __ldg(bias + c * 32 + j);
          const float a = fmaxf(v0[j] + bj, 0.f), d = fmaxf(v1[j] + bj, 0.f);
          // scan order of the 2x2 window: (row 0, x even)=0, (row 0, x odd)=1, (row 1, even)=2, (row 1, odd)=3;
          // the first maximum wins: larger value, ties to the smaller index
          float vs = a; uint32_t ks = (uint32_t)odd;
          if (d > a) { vs = d; ks = 2u + (uint32_t)odd; }
          const float vo = __shfl_xor_sync(0xffffffffu, vs, 1);
          const uint32_t ko = __shfl_xor_sync(0xffffffffu, ks, 1);
          const bool other = vo > vs || (vo == vs && ko < ks);
          const float mv = other ? vo : vs;
          const uint32_t mk = other ? ko : ks;
          m[j] = mv;
          code[j >> 3] |= (mv > 0.f ? mk : 4u) << (3 * (j & 7));
        }
        // both lanes of a pair hold the pooled pixel: the even lane stores channels 0-15 of this chunk, the odd 16-31
        uint32_t pk[8];
#pragma unroll
        for (int h = 0; h < 8; ++h) {
          const __nv_bfloat162 p = __floats2bfloat162_rn(odd ? m[16 + 2 * h] : m[2 * h], odd ? m[17 + 2 * h] : m[2 * h + 1]);
          pk[h] = *reinterpret_cast<const uint32_t*>(&p);
        }
        uint4* op = reinterpret_cast<uint4*>(prow + c * 32 + odd * 16);
        op[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
        op[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
        *reinterpret_cast<uint2*>(crow + c * 4 + odd * 2) = odd ? make_uint2(code[2], code[3]) : make_uint2(code[0], code[1]);
      } else if (TMA_EPI) {
        // Both warps of a quarter fill their halves of the quarter's 32 x 128 B staging block, meet at a 64-thread named
        // barrier, and one lane issues the TMA store of the block.
        const int q0w0 = ROWS ? ((item / (g.H >> 1)) * g.Hp + 2 * (item % (g.H >> 1)) + 1) * g.Wp + 1 + ew * 32 : item * T * 128 + ew * 32;
        const int qstep = ROWS ? g.Wp : 128;
#pragma unroll 1
        for (int t = 0; t < T; ++t) {
          const int q0w = q0w0 + t * qstep;
          const int q = q0w + lane;
          const int n = q / HpWp, rem = q - n * HpWp;
          const int yp = rem / g.Wp, xp = rem - yp * g.Wp;
          const bool valid = q < g.Q && xp >= 1 && xp <= g.W && yp >= 1 && yp <= g.H;
          const size_t o_f32 = (((size_t)n * g.H + (yp - 1)) * g.W + (xp - 1)) * N_OUT;
          uint32_t mo[N_OUT / 64];                  // own chunk of each 64-channel half
#pragma unroll
          for (int hf = 0; hf < N_OUT / 64; ++hf) {
            const int c = hf * 2 + eg;
            float v[32];
            wg_sync(); stage_acc64(acc, t * (N_OUT / 64) + hf, stg); wg_sync();
            stg_read32(stg, erow, eg * 32, v);
            if (bias) {
#pragma unroll
              for (int j = 0; j < 32; j += 4) {
                const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + c * 32 + j));
                v[j] += bv.x; v[j + 1] += bv.y; v[j + 2] += bv.z; v[j + 3] += bv.w;
              }
            }
            if (relu) {
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
            }
            if (mask_bits) {
              const uint32_t w = t ? mbt[1][c] : mbt[0][c];
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] = ((w >> j) & 1u) ? v[j] : 0.f;
            }
            mo[hf] = 0u;
            if (mask_out) {
              uint32_t w = 0;
#pragma unroll
              for (int j = 0; j < 32; ++j) w |= (v[j] > 0.f ? 1u : 0u) << j;
              mo[hf] = w;
            }
            // the staging block may still be read by the previous TMA store: wait right before the first write
            if (store_pending) { if (issuer) bulk_wait_read0(); pair_sync(); store_pending = false; }
#pragma unroll
            for (int j4 = 0; j4 < 4; ++j4) {
              const uint32_t addr = my_row + (uint32_t)(((eg * 4 + j4) ^ sw) << 4);
              uint4 pk = make_uint4(0, 0, 0, 0);                               // border / out-of-range positions store zeros
              if (valid) {
                __nv_bfloat162 p0 = __floats2bfloat162_rn(v[j4 * 8 + 0], v[j4 * 8 + 1]);
                __nv_bfloat162 p1 = __floats2bfloat162_rn(v[j4 * 8 + 2], v[j4 * 8 + 3]);
                __nv_bfloat162 p2 = __floats2bfloat162_rn(v[j4 * 8 + 4], v[j4 * 8 + 5]);
                __nv_bfloat162 p3 = __floats2bfloat162_rn(v[j4 * 8 + 6], v[j4 * 8 + 7]);
                pk.x = *reinterpret_cast<uint32_t*>(&p0); pk.y = *reinterpret_cast<uint32_t*>(&p1);
                pk.z = *reinterpret_cast<uint32_t*>(&p2); pk.w = *reinterpret_cast<uint32_t*>(&p3);
              }
              asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(pk.x), "r"(pk.y), "r"(pk.z), "r"(pk.w) : "memory");
            }
            if (out_f32 && valid) {
              float4* fp = reinterpret_cast<float4*>(out_f32 + o_f32 + c * 32);
#pragma unroll
              for (int j = 0; j < 8; ++j) fp[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
            }
            fence_proxy_async();                    // generic-proxy smem writes -> visible to the TMA engine
            pair_sync();                            // both 64-byte halves of every row are in place
            if (issuer && q0w < g.Q) { tma_store_2d(&tmOut, estg, hf * 64, q0w); bulk_commit(); }
            store_pending = true;
          }
          if (mask_out && q < g.Q) {
#pragma unroll
            for (int hf = 0; hf < N_OUT / 64; ++hf) mask_out[(size_t)q * (N_OUT / 32) + hf * 2 + eg] = valid ? mo[hf] : 0u;
          }
        }
      } else {
#pragma unroll 1
        for (int t = 0; t < T; ++t) {
          const int q = (ROWS ? ((item / (g.H >> 1)) * g.Hp + 2 * (item % (g.H >> 1)) + 1 + t) * g.Wp + 1 : (item * T + t) * 128) + ew * 32 + lane;
          const int n = q / HpWp, rem = q - n * HpWp;
          const int yp = rem / g.Wp, xp = rem - yp * g.Wp;
          const bool valid = q < g.Q && xp >= 1 && xp <= g.W && yp >= 1 && yp <= g.H;
          const size_t o_pad = (size_t)q * N_OUT;
          const size_t o_f32 = (((size_t)n * g.H + (yp - 1)) * g.W + (xp - 1)) * N_OUT;
#pragma unroll
          for (int hf = 0; hf < N_OUT / 64; ++hf) {
            const int c = hf * 2 + eg;
            float v[32];
            wg_sync(); stage_acc64(acc, t * (N_OUT / 64) + hf, stg); wg_sync();
            stg_read32(stg, erow, eg * 32, v);
            if (valid) {
              if (bias) {
#pragma unroll
                for (int j = 0; j < 32; j += 4) {
                  const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + c * 32 + j));
                  v[j] += bv.x; v[j + 1] += bv.y; v[j + 2] += bv.z; v[j + 3] += bv.w;
                }
              }
              if (relu) {
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
              }
              if (mask_bits) {
                const uint32_t w = __ldg(mask_bits + (size_t)q * (N_OUT / 32) + c);
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = ((w >> j) & 1u) ? v[j] : 0.f;
              }
              if (mask_out) {
                uint32_t w = 0;
#pragma unroll
                for (int j = 0; j < 32; ++j) w |= (v[j] > 0.f ? 1u : 0u) << j;
                mask_out[(size_t)q * (N_OUT / 32) + c] = w;
              }
              if (mask_src) {
                const uint4* mp = reinterpret_cast<const uint4*>(mask_src + o_pad + c * 32);
#pragma unroll
                for (int j4 = 0; j4 < 4; ++j4) {
                  const uint4 m = __ldg(mp + j4);
                  const uint32_t mw[4] = {m.x, m.y, m.z, m.w};
#pragma unroll
                  for (int h = 0; h < 4; ++h) {
                    // bf16 > 0  <=>  sign bit clear and magnitude non-zero
                    const uint32_t lo = mw[h] & 0xFFFFu, hi = mw[h] >> 16;
                    if (!(lo != 0 && !(lo & 0x8000u))) v[j4 * 8 + h * 2] = 0.f;
                    if (!(hi != 0 && !(hi & 0x8000u))) v[j4 * 8 + h * 2 + 1] = 0.f;
                  }
                }
              }
              if (out_bf) {
                uint4* op = reinterpret_cast<uint4*>(out_bf + o_pad + c * 32);
#pragma unroll
                for (int j4 = 0; j4 < 4; ++j4) {
                  uint4 pk;
                  __nv_bfloat162 p0 = __floats2bfloat162_rn(v[j4 * 8 + 0], v[j4 * 8 + 1]);
                  __nv_bfloat162 p1 = __floats2bfloat162_rn(v[j4 * 8 + 2], v[j4 * 8 + 3]);
                  __nv_bfloat162 p2 = __floats2bfloat162_rn(v[j4 * 8 + 4], v[j4 * 8 + 5]);
                  __nv_bfloat162 p3 = __floats2bfloat162_rn(v[j4 * 8 + 6], v[j4 * 8 + 7]);
                  pk.x = *reinterpret_cast<uint32_t*>(&p0); pk.y = *reinterpret_cast<uint32_t*>(&p1);
                  pk.z = *reinterpret_cast<uint32_t*>(&p2); pk.w = *reinterpret_cast<uint32_t*>(&p3);
                  op[j4] = pk;
                }
              }
              if (out_f32) {
                float4* fp = reinterpret_cast<float4*>(out_f32 + o_f32 + c * 32);
#pragma unroll
                for (int j = 0; j < 8; ++j) fp[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
              }
            }
          }
        }
      }
    }
    if (TMA_EPI && issuer) bulk_wait0();
    __syncwarp();
  }
}

}  // namespace tc
}  // namespace udh
