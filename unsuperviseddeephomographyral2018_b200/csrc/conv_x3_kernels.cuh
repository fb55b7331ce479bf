// Error-compensated wgmma implicit-GEMM 3x3 convolution (UDH_NUMERIC_BF16X3): fp32-grade results from 16-bit tensor-core
// operands.  Same padded-stream formulation as conv_tc_kernels.cuh (every tap is a row shift of the flattened activation
// matrix), but every fp32 value travels as TWO 16-bit limbs, x = hi + lo:
//   * activation / gradient streams are [Q positions][hi(C) | lo(C)], packed weights hold [tap][cb][hi | lo][N][64];
//   * a product is evaluated as  lo_x.hi_w + hi_x.hi_w + hi_x.lo_w  — three wgmma passes into ONE fp32 register
//     accumulator (the dropped lo.lo term and the residual of the split are 2^-16 relative for bf16 limbs);
//   * the epilogue applies bias / ReLU / ReLU-backward mask on the fp32 accumulator, splits the result into limbs again and
//     TMA-stores both (so rounding to 16 bits never enters the data path: the only approximation is the 2^-16 split).
// Shared memory cannot hold double-buffered operands of twice the size, so the two limbs of the A rows live in two SINGLE
// buffers that are consumed in staggered phases: phase LO (A_lo x W_hi, 1/3 of the MMAs) then phase HI (A_hi x W_hi,
// A_hi x W_lo).  A_lo is free again after a third of the item and is refilled under phase HI; A_hi is refilled under the
// next item's phase LO — each limb buffer has its own full/empty mbarrier pair, and a dedicated producer warp so that the
// weight ring (a second producer warp) never waits behind an activation buffer.  Weights always stream through a TMA ring
// (hi + lo of all 9 taps do not fit next to the activations); each ring block is reused by the T tiles of the item.
//   warpgroup 0: weight-ring producer (warp 0), activation producer (warp 3) | warpgroups 1-2: MMA + epilogue, each owning
//   64 of the 128 rows of every tile (accumulators in registers, drained through stage_acc32 as in the bf16 kernel).
// Phase order: HI first (its first MMA initialises the accumulators), then LO.
// WIDE (64 -> 64 channels): phase HI issues ONE N = 128 MMA per k-step against the ring stage [W_hi | W_lo] into a MAIN and
// an AUX accumulator (adjacent columns of one fragment) instead of two N = 64 MMAs; phase LO adds A_lo x W_hi into MAIN;
// the epilogue reads MAIN + AUX.
#pragma once
#include "conv_tc_kernels.cuh"

namespace udh {
namespace tc {

constexpr int kX3MaxStages = 6;

template <int N_OUT, int CB, int T, bool WIDE = false>
struct ConvX3Smem {
  static constexpr int kWStageBytes = N_OUT * 128 * (WIDE ? 2 : 1);
  // fixed part: alignment slack + both limbs of the A rows + epilogue staging + accumulator transpose blocks + barriers
  static size_t fixed_bytes(int abuf_rows) { return 1024 + (size_t)2 * CB * abuf_rows * 128 + kEpiStageBytes + 2 * kStg32Bytes + 256; }
  static int stages(int abuf_rows) {
    const long long left = 232448ll - (long long)fixed_bytes(abuf_rows);
    const int s = (int)(left / kWStageBytes);
    return s > kX3MaxStages ? kX3MaxStages : s;
  }
};

// The weight ring has `stages` slots (a runtime value: as many as shared memory holds next to the activation rows).
// ROWS (W == 128 images, 64 -> 64 channels, T == 2, not WIDE: conv1_2).  An item is the interior of two consecutive image rows
// (2y, 2y+1): tile t starts at the first interior position of row 2y + t, i.e. the tiles are Wp (not 128) positions apart in
// the same staged rows, no border position is computed, and the epilogue thread of column x holds both rows of that column.
//   ROWS == 1: forward fused with the 2x2 max-pool — bias + ReLU, maximum (vertical in registers, horizontal with one lane
//              exchange), then the POOLED two-limb stream and the 3-bit routing codes of the max-pool backward are written; the
//              full-resolution activation (554 MB in this mode) is never written or re-read;
//   ROWS == 2: the ordinary epilogue (bias / ReLU-backward mask / limb split / TMA store) on row tiles (the dgrad).
template <int N_OUT, int CB, int T, int FMT_A, int FMT_W, int FMT_O, bool WIDE = false, int ROWS = 0>
__global__ void __launch_bounds__(384, 1)
tc_conv_x3_kernel(const __grid_constant__ CUtensorMap tmA128, const __grid_constant__ CUtensorMap tmAhh,
                  const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmOut, const ConvGeom g,
                  const int stages, const float* __restrict__ bias, const uint32_t* __restrict__ mask_bits,
                  uint32_t* __restrict__ mask_out, float* __restrict__ out_f32, const int relu, const float out_scale) {
  static_assert(FMT_A == kFmtBF16 && FMT_W == kFmtBF16, "wgmma multiplies limbs of one format");
  extern __shared__ uint8_t raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~(uintptr_t)1023);
  const int abuf_bytes = g.abuf_rows * 128;                       // one 64-channel block of one limb
  uint8_t* sA = base;                                             // [2 limbs][CB][abuf_rows][128]
  uint8_t* sW = base + (size_t)2 * CB * abuf_bytes;               // [stages][N_OUT][128]
  static_assert(!WIDE || (N_OUT == 64 && T <= 2), "WIDE: 64 output channels, two accumulators per tile");
  static_assert(ROWS == 0 || (N_OUT == 64 && CB == 1 && T == 2), "row tiles: the 64-channel instance with two tiles");
  constexpr bool POOL = ROWS == 1;
  // first position of an item and distance between its tiles (in positions)
  auto item_q0 = [&](int item) { return ROWS ? ((item / (g.H >> 1)) * g.Hp + 2 * (item % (g.H >> 1)) + 1) * g.Wp + 1 : item * T * 128; };
  const int tstep = ROWS ? g.Wp : 128;
  constexpr int kAcc = WIDE ? 2 : 1;                              // accumulators per tile (MAIN | AUX)
  constexpr int kTileCols = N_OUT * kAcc;                         // accumulator columns per tile
  constexpr int kTileRegs = kTileCols / 2;                        // fragment registers per tile
  constexpr int kStageBytes = N_OUT * 128 * kAcc;                 // one ring stage: [W_hi] or [W_hi | W_lo]
  uint8_t* sEpi = sW + (size_t)stages * kStageBytes;              // [4 quarters][32 rows][128 B]
  float* sStg = reinterpret_cast<float*>(sEpi + kEpiStageBytes);  // [2 warpgroups][kStg32Bytes]
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sStg) + 2 * kStg32Bytes);
  uint64_t* a_full = bars;            // [2] per limb (0 = hi, 1 = lo)
  uint64_t* a_empty = bars + 2;       // [2]
  uint64_t* w_full = bars + 4;        // [kX3MaxStages]
  uint64_t* w_empty = bars + 4 + kX3MaxStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  static_assert(T <= 4, "mask prefetch registers are sized for T <= 4");

  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], 256); }
    for (int i = 0; i < kX3MaxStages; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], 256); }
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) { prefetch_tmap(&tmW); prefetch_tmap(&tmOut); }
  if (warp == 3 && lane == 0) { prefetch_tmap(&tmA128); prefetch_tmap(&tmAhh); }
  __syncthreads();
  const int my_items = (g.num_items - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // items blockIdx.x + i*gridDim.x
  pdl_wait();                  // predecessor grid complete: global memory may be touched from here on
  pdl_trigger();

  if (warp < 4) {
    regs_dec<40>();
    if (warp == 3 && lane == 0) {
      // ===================================== activation producer =====================================
      for (int it = 0; it < my_items; ++it) {
        const int q0 = item_q0((int)blockIdx.x + it * (int)gridDim.x);
#pragma unroll 1
        for (int l = 0; l < 2; ++l) {                             // consumption order: hi limb first
          mbar_wait(&a_empty[l], (it & 1) ^ 1);
          mbar_arrive_expect_tx(&a_full[l], (uint32_t)(CB * abuf_bytes));
          for (int cb = 0; cb < CB; ++cb) {
            uint8_t* dst = sA + (size_t)(l * CB + cb) * abuf_bytes;
            const int c0 = (l * CB + cb) * 64;                    // channel coordinate in the [hi | lo] stream
            tma_load_2d(dst, &tmAhh, c0, q0 - g.hh, &a_full[l]);
            for (int t = 0; t < T; ++t)
              tma_load_2d(dst + (size_t)(g.hh + t * 128) * 128, &tmA128, c0, q0 + t * 128, &a_full[l]);
            tma_load_2d(dst + (size_t)(g.hh + T * 128) * 128, &tmAhh, c0, q0 + T * 128, &a_full[l]);
          }
        }
      }
    } else if (warp == 0 && lane == 0) {
      // ===================================== weight-ring producer =====================================
      uint32_t ws = 0, wpar = 1;                                  // first pass over the ring: the slots are free
      auto push = [&](int block, int nblocks) {                  // `nblocks` consecutive [N_OUT][64] blocks into one stage
        mbar_wait(&w_empty[ws], wpar);
        mbar_arrive_expect_tx(&w_full[ws], (uint32_t)(nblocks * N_OUT * 128));
        for (int i = 0; i < nblocks; ++i)
          tma_load_2d(sW + (size_t)ws * kStageBytes + (size_t)i * N_OUT * 128, &tmW, 0, (block + i) * N_OUT, &w_full[ws]);
        if (++ws == (uint32_t)stages) { ws = 0; wpar ^= 1u; }
      };
      for (int it = 0; it < my_items; ++it) {
        for (int kb = 0; kb < 9 * CB; ++kb) {                                     // phase HI: A_hi x W_hi, A_hi x W_lo
          if (WIDE) push(kb * 2, 2);
          else { push(kb * 2, 1); push(kb * 2 + 1, 1); }
        }
        for (int kb = 0; kb < 9 * CB; ++kb) push(kb * 2, 1);                      // phase LO: A_lo x W_hi
      }
    }
  } else {
    regs_inc<232>();
    const int cw = (warp - 4) >> 2;               // MMA warpgroup: rows [64 cw, 64 cw + 64) of every tile
    const int wi = warp & 3;
    const int ew = 2 * cw + (wi & 1);             // row quarter of the tile this warp drains
    const int eg = wi >> 1;                       // 32-column chunk parity this warp drains
    const int erow = 32 * (wi & 1) + lane;
    float* stg = sStg + cw * (kStg32Bytes / 4);
    auto wg_sync = [&]() { named_sync(5 + cw, 128); };
    const uint32_t a_addr0 = smem_u32(sA) + (uint32_t)cw * 64 * 128, w_addr0 = smem_u32(sW);
    const uint32_t w_stage_units = (uint32_t)kStageBytes >> 4;
    const uint32_t w_lo0 = desc_lo(w_addr0, 16);
    const uint32_t cb_units = (uint32_t)abuf_bytes >> 4;
    const uint32_t wp8 = (uint32_t)g.Wp * 8;                      // one image row of taps, in sixteen-byte units
    uint32_t ws = 0, wpar = 0;
    float acc[T * kTileRegs];
    // 32 columns (block b32 of the fragment) of row erow of the warpgroup, for the warps of chunk parity eg; every warp
    // of the warpgroup takes part (two transpose rounds, one per parity)
    auto fetch = [&](int b32, float (&v)[32]) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        wg_sync(); stage_acc32(acc, b32 + e, stg); wg_sync();
        if (e == eg) stg32_read32(stg, erow, v);
      }
    };
    const int HpWp = g.Hp * g.Wp;
    uint8_t* estg = sEpi + ew * 4096;
    const uint32_t my_row = smem_u32(estg) + lane * 128;
    const int sw = lane & 7;
    const bool issuer = eg == 0 && lane == 0;
    auto pair_sync = [&]() { named_sync(1 + ew, 64); };
    bool store_pending = false;
    for (int it = 0; it < my_items; ++it) {
      const int item = (int)blockIdx.x + it * (int)gridDim.x;
      const int q0w0 = item_q0(item) + ew * 32;
      // ReLU-backward mask words (1 bit / element) of all T tiles, requested before the MMAs
      uint32_t mbt[T][2];
      if (!POOL) {
#pragma unroll
        for (int t = 0; t < T; ++t) {
          const int qt = q0w0 + t * tstep + lane;
          const bool ok = mask_bits && qt < g.Q;
          if (N_OUT == 64) {
            mbt[t][0] = ok ? __ldg(mask_bits + (size_t)qt * 2 + eg) : 0u; mbt[t][1] = 0u;
          } else {
            mbt[t][0] = ok ? __ldg(mask_bits + (size_t)qt * 4 + eg) : 0u;
            mbt[t][1] = ok ? __ldg(mask_bits + (size_t)qt * 4 + 2 + eg) : 0u;
          }
        }
      }
      // ===================================== MMA =====================================
      acc_fence(acc);
      int prev = -1;
      bool first = true;                                          // the very first MMA of the item overwrites the accumulators
#pragma unroll 1
      for (int ph = 0; ph < 2; ++ph) {                            // phase 0 consumes the hi limb, phase 1 the lo limb
        mbar_wait(&a_full[ph], it & 1);
        // descriptor (low word) of tap (0,0), channel block 0 of this limb: rows start at hh - Wp - 1
        const uint32_t a_tap0 = desc_lo(a_addr0 + (uint32_t)(ph * CB) * abuf_bytes + (uint32_t)(g.hh - g.Wp - 1) * 128, 16);
#pragma unroll 1
        for (int kb = 0; kb < 9 * CB; ++kb) {
          const int tap = kb / CB, cb = kb - tap * CB;
          const int ky = tap / 3, kx = tap - ky * 3;
          const uint32_t a_lo = a_tap0 + (uint32_t)ky * wp8 + (uint32_t)(kx * 8) + (uint32_t)cb * cb_units;
#pragma unroll
          for (int wl = 0; wl < 2; ++wl) {
            if (wl == 1 && (ph == 1 || WIDE)) continue;           // phase LO multiplies with W_hi only; WIDE: one [hi | lo] stage
            mbar_wait(&w_full[ws], wpar);
            const uint32_t w_lo = w_lo0 + ws * w_stage_units;
            wg_fence();
#pragma unroll
            for (int t = 0; t < T; ++t) {
              float (&d)[kTileRegs] = *reinterpret_cast<float(*)[kTileRegs]>(&acc[t * kTileRegs]);
              const uint32_t a_t = a_lo + (ROWS ? (uint32_t)t * wp8 : (uint32_t)(t * 1024));
#pragma unroll
              for (int k = 0; k < 4; ++k) {     // +2 sixteen-byte units per 32-byte k-step
                const uint32_t accum = (first && k == 0) ? 0u : 1u;
                if constexpr (WIDE) {
                  if (ph == 0) wgmma_bf16_head<2 * N_OUT, 0, 0>(d, desc_from_lo(a_t + k * 2), desc_from_lo(w_lo + k * 2), accum);
                  else wgmma_bf16_head<N_OUT, 0, 0>(d, desc_from_lo(a_t + k * 2), desc_from_lo(w_lo + k * 2), accum);
                } else {
                  wgmma_bf16_head<N_OUT, 0, 0>(d, desc_from_lo(a_t + k * 2), desc_from_lo(w_lo + k * 2), accum);
                }
              }
            }
            wg_commit();
            wg_wait<1>();                                         // the previous stage's MMAs are done: its slot is free
            if (prev >= 0) mbar_arrive(&w_empty[prev]);
            prev = (int)ws;
            first = false;
            if (++ws == (uint32_t)stages) { ws = 0; wpar ^= 1u; }
          }
        }
        wg_wait<0>();
        mbar_arrive(&w_empty[prev]);
        prev = -1;
        mbar_arrive(&a_empty[ph]);                                // this limb's rows are no longer read -> producer
      }
      acc_fence(acc);
      // ===================================== epilogue =====================================
      if constexpr (POOL) {
        // thread = image column x (W == 128 == tile rows); warps of parity eg pool the 32-channel chunk eg
        const int OH = g.H >> 1, OW = g.W >> 1;
        const int x = ew * 32 + lane;
        const int px = x >> 1, odd = x & 1;
        uint16_t* out_pool = reinterpret_cast<uint16_t*>(out_f32);             // pooled two-limb stream [B][OH+2][OW+2][hi 64 | lo 64]
        const int n = item / OH, yy = item - n * OH;
        uint16_t* prow = out_pool + (((size_t)n * (OH + 2) + yy + 1) * (OW + 2) + px + 1) * 128;
        uint32_t* crow = mask_out + (((size_t)n * OH + yy) * OW + px) * 8;
        const int c = eg;
        float v0[32], v1[32], u[32];
        fetch(0, v0);                                             // tile 0 (+ AUX)
        if (WIDE) {
          fetch(2, u);
#pragma unroll
          for (int j = 0; j < 32; ++j) v0[j] += u[j];
        }
        fetch(kTileCols / 32, v1);                                // tile 1 (+ AUX)
        if (WIDE) {
          fetch(kTileCols / 32 + 2, u);
#pragma unroll
          for (int j = 0; j < 32; ++j) v1[j] += u[j];
        }
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
        uint32_t ph_[8], pl_[8];
#pragma unroll
        for (int h = 0; h < 8; ++h) split2<FMT_O>(odd ? m[16 + 2 * h] : m[2 * h], odd ? m[17 + 2 * h] : m[2 * h + 1], ph_[h], pl_[h]);
        uint4* oh = reinterpret_cast<uint4*>(prow + c * 32 + odd * 16);
        oh[0] = make_uint4(ph_[0], ph_[1], ph_[2], ph_[3]); oh[1] = make_uint4(ph_[4], ph_[5], ph_[6], ph_[7]);
        uint4* ol = reinterpret_cast<uint4*>(prow + 64 + c * 32 + odd * 16);
        ol[0] = make_uint4(pl_[0], pl_[1], pl_[2], pl_[3]); ol[1] = make_uint4(pl_[4], pl_[5], pl_[6], pl_[7]);
        *reinterpret_cast<uint2*>(crow + c * 4 + odd * 2) = odd ? make_uint2(code[2], code[3]) : make_uint2(code[0], code[1]);
      } else {
        // Both warps of a quarter fill their halves of the quarter's 32 x 128 B staging block, meet at a 64-thread named
        // barrier, and one lane issues the TMA store; the hi block and the lo block of a half go through the same block.
#pragma unroll 1
        for (int t = 0; t < T; ++t) {
          const int q0w = q0w0 + t * tstep;
          const int q = q0w + lane;
          const int n = q / HpWp, rem = q - n * HpWp;
          const int yp = rem / g.Wp, xp = rem - yp * g.Wp;
          const bool valid = q < g.Q && xp >= 1 && xp <= g.W && yp >= 1 && yp <= g.H;
          const size_t o_f32 = (((size_t)n * g.H + (yp - 1)) * g.W + (xp - 1)) * N_OUT;
          uint32_t mo[N_OUT / 64];
#pragma unroll
          for (int hf = 0; hf < N_OUT / 64; ++hf) {
            const int c = hf * 2 + eg;
            float v[32];
            fetch(t * (kTileCols / 32) + hf * 2, v);
            if (WIDE) {                                           // MAIN (A.W_hi terms) + AUX (A_hi.W_lo)
              float u[32];
              fetch(t * (kTileCols / 32) + N_OUT / 32 + hf * 2, u);
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] += u[j];
            }
            if (out_scale != 1.0f) {
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] *= out_scale;
            }
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
              const uint32_t w = mbt[t][hf];
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
            uint32_t hi[16], lo[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              if (valid) split2<FMT_O>(v[2 * j], v[2 * j + 1], hi[j], lo[j]);
              else { hi[j] = 0u; lo[j] = 0u; }                       // border / out-of-range positions store zeros
            }
#pragma unroll
            for (int limb = 0; limb < 2; ++limb) {
              // the staging block may still be read by the previous TMA store
              if (store_pending) { if (issuer) bulk_wait_read0(); pair_sync(); }
#pragma unroll
              for (int j4 = 0; j4 < 4; ++j4) {
                const uint32_t addr = my_row + (uint32_t)(((eg * 4 + j4) ^ sw) << 4);
                const uint32_t* src = limb ? lo : hi;
                asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(src[j4 * 4]), "r"(src[j4 * 4 + 1]),
                             "r"(src[j4 * 4 + 2]), "r"(src[j4 * 4 + 3]) : "memory");
              }
              fence_proxy_async();                    // generic-proxy smem writes -> visible to the TMA engine
              pair_sync();                            // both 64-byte halves of every row are in place
              if (issuer && q0w < g.Q) { tma_store_2d(&tmOut, estg, limb * N_OUT + hf * 64, q0w); bulk_commit(); }
              store_pending = true;
            }
            if (out_f32 && valid) {
              float4* fp = reinterpret_cast<float4*>(out_f32 + o_f32 + c * 32);
#pragma unroll
              for (int j = 0; j < 8; ++j) fp[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
            }
          }
          if (mask_out && q < g.Q) {
#pragma unroll
            for (int hf = 0; hf < N_OUT / 64; ++hf) mask_out[(size_t)q * (N_OUT / 32) + hf * 2 + eg] = valid ? mo[hf] : 0u;
          }
        }
      }
    }
    if (!POOL && issuer) bulk_wait0();
    __syncwarp();
  }
}

}  // namespace tc
}  // namespace udh
