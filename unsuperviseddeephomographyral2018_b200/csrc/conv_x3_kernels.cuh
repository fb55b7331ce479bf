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
//   warpgroup 0: weight-ring producer (warp 0), activation producer (warp 3) | warpgroups 1-2: MMA | warpgroup 3: epilogue.
// Phase order: HI first (its first MMA initialises the accumulators), then LO.
// 128 output channels: each MMA warpgroup owns 64 of the 128 rows of every tile, D[pos][co] = X . W with the activation
// rows as A and the ring stage as B (m64n128k16).
// 64 output channels (TR): the tile is transposed, D^T[co][pos] = W . X^T: the ring stage [64 co][64 ci] is the A operand
// and 128 activation rows are the B operand, so each MMA is an m64n128k16 (2 KB + 4 KB of shared memory per 131 072 MACs)
// instead of two m64n64k16 (4 KB + 4 KB); at N = 64 the operand reads alone would need all 128 B/clk of shared memory at
// tensor peak.  MMA warpgroup cw owns the whole tile t = cw.  Every output element sees the same chain of k16 partial
// products as in the untransposed tile (same stages, same k-step order, same first / accumulate flags).  The epilogue
// warpgroup reads the fragment column-wise out of the shared-memory handoff so that, as for 128 channels, one thread works
// on 32 channels of one position.
#pragma once
#include "conv_tc_kernels.cuh"

namespace udh {
namespace tc {

constexpr int kX3MaxStages = 6;

// v[j] = 32 consecutive fp32 at shared address addr (part of a handoff row)
__device__ __forceinline__ void lds_read32(uint32_t addr, float (&v)[32]) {
#pragma unroll
  for (int j = 0; j < 8; ++j)
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v[4 * j]), "=f"(v[4 * j + 1]), "=f"(v[4 * j + 2]), "=f"(v[4 * j + 3])
                 : "r"(addr + 16 * j) : "memory");
}

// The weight ring has `stages` slots (a runtime value: as many as shared memory holds next to the activation rows).
// ROWS (W == 128 images, 64 -> 64 channels, T == 2: conv1_2).  An item is the interior of two consecutive image rows
// (2y, 2y+1): tile t starts at the first interior position of row 2y + t, i.e. the tiles are Wp (not 128) positions apart in
// the same staged rows, and no border position is computed.
//   ROWS == 1: forward fused with the 2x2 max-pool — the epilogue thread of column x reads that column of both rows; bias +
//              ReLU, maximum (vertical in registers, horizontal with one lane exchange), then the POOLED two-limb stream and
//              the 3-bit routing codes of the max-pool backward are written; the full-resolution activation (554 MB in this
//              mode) is never written or re-read;
//   ROWS == 2: the ordinary epilogue (bias / ReLU-backward mask / limb split / TMA store) on row tiles (the dgrad).

// first position of an item and distance between its tiles (in positions)
template <int T, int ROWS>
__device__ __forceinline__ int x3_item_q0(const ConvGeom& g, int item) {
  return ROWS ? ((item / (g.H >> 1)) * g.Hp + 2 * (item % (g.H >> 1)) + 1) * g.Wp + 1 : item * T * 128;
}

// activation producer (one thread): both limbs of the A rows of every item, hi limb first (the consumption order).
// lo_free: the epilogue's h_empty, whose phase must also complete before the lo buffer of the next item is loaded (the
// handoff lives in that buffer).  The kernel always passes it; the null test stays because without it ptxas allocates
// registers differently in every instance.
template <int CB, int T, int ROWS>
__device__ __forceinline__ void x3_produce_acts(const CUtensorMap* tmA128, const CUtensorMap* tmAhh, const ConvGeom& g, int my_items,
                                                uint8_t* sA, uint64_t* a_full, uint64_t* a_empty, uint64_t* lo_free) {
  const int abuf_bytes = g.abuf_rows * 128;
  for (int it = 0; it < my_items; ++it) {
    const int q0 = x3_item_q0<T, ROWS>(g, (int)blockIdx.x + it * (int)gridDim.x);
#pragma unroll 1
    for (int l = 0; l < 2; ++l) {
      mbar_wait(&a_empty[l], (it & 1) ^ 1);
      if (l == 1 && lo_free) mbar_wait(lo_free, (it & 1) ^ 1);
      mbar_arrive_expect_tx(&a_full[l], (uint32_t)(CB * abuf_bytes));
      for (int cb = 0; cb < CB; ++cb) {
        uint8_t* dst = sA + (size_t)(l * CB + cb) * abuf_bytes;
        const int c0 = (l * CB + cb) * 64;                        // channel coordinate in the [hi | lo] stream
        tma_load_2d(dst, tmAhh, c0, q0 - g.hh, &a_full[l]);
        for (int t = 0; t < T; ++t)
          tma_load_2d(dst + (size_t)(g.hh + t * 128) * 128, tmA128, c0, q0 + t * 128, &a_full[l]);
        tma_load_2d(dst + (size_t)(g.hh + T * 128) * 128, tmAhh, c0, q0 + T * 128, &a_full[l]);
      }
    }
  }
}

// weight-ring producer (one thread): per item, phase HI's blocks (A_hi x W_hi, A_hi x W_lo) then phase LO's (A_lo x W_hi)
template <int N_OUT, int CB>
__device__ __forceinline__ void x3_produce_weights(const CUtensorMap* tmW, int my_items, int stages, uint8_t* sW, uint64_t* w_full,
                                                   uint64_t* w_empty) {
  constexpr int kStageBytes = N_OUT * 128;
  uint32_t ws = 0, wpar = 1;                                      // first pass over the ring: the slots are free
  auto push = [&](int block) {                                    // one [N_OUT][64] block into one stage
    mbar_wait(&w_empty[ws], wpar);
    mbar_arrive_expect_tx(&w_full[ws], (uint32_t)kStageBytes);
    tma_load_2d(sW + (size_t)ws * kStageBytes, tmW, 0, block * N_OUT, &w_full[ws]);
    if (++ws == (uint32_t)stages) { ws = 0; wpar ^= 1u; }
  };
  for (int it = 0; it < my_items; ++it) {
    for (int kb = 0; kb < 9 * CB; ++kb) { push(kb * 2); push(kb * 2 + 1); }
    for (int kb = 0; kb < 9 * CB; ++kb) push(kb * 2);
  }
}

// The MMAs of one item for one MMA warpgroup, into acc (T tiles; TR: the warpgroup's transposed tile).  a_addr0: shared
// address of this warpgroup's first A row in the hi buffer; ws / wpar: ring position, carried from item to item.  Each limb
// buffer is released (a_empty) once this warpgroup's last MMA reading it has completed.
template <int N_OUT, int CB, int T>
__device__ __forceinline__ void x3_mma_item(float (&acc)[T * N_OUT / 2], int it, const ConvGeom& g, int stages, uint32_t a_addr0,
                                            uint32_t w_lo0, uint64_t* a_full, uint64_t* a_empty, uint64_t* w_full, uint64_t* w_empty,
                                            uint32_t& ws, uint32_t& wpar) {
  constexpr bool TR = N_OUT == 64;
  constexpr int kTileRegs = N_OUT / 2;
  const uint32_t abuf_bytes = (uint32_t)g.abuf_rows * 128;
  const uint32_t w_stage_units = (uint32_t)(N_OUT * 128) >> 4;
  const uint32_t cb_units = abuf_bytes >> 4;
  const uint32_t wp8 = (uint32_t)g.Wp * 8;                        // one image row of taps, in sixteen-byte units
  acc_fence(acc);
  int prev = -1;
  bool first = true;                                              // the very first MMA of the item overwrites the accumulators
#pragma unroll 1
  for (int ph = 0; ph < 2; ++ph) {                                // phase 0 consumes the hi limb, phase 1 the lo limb
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
        if (wl == 1 && ph == 1) continue;                         // phase LO multiplies with W_hi only
        mbar_wait(&w_full[ws], wpar);
        const uint32_t w_lo = w_lo0 + ws * w_stage_units;
        wg_fence();
        if constexpr (TR) {
#pragma unroll
          for (int k = 0; k < 4; ++k)           // +2 sixteen-byte units per 32-byte k-step; A = weights, B = activation rows
            wgmma_bf16<128, 0, 0>(acc, desc_from_lo(w_lo + k * 2), desc_from_lo(a_lo + k * 2), (first && k == 0) ? 0u : 1u);
        } else {
#pragma unroll
          for (int t = 0; t < T; ++t) {
            float (&d)[kTileRegs] = *reinterpret_cast<float(*)[kTileRegs]>(&acc[t * kTileRegs]);
            const uint32_t a_t = a_lo + (uint32_t)(t * 1024);
#pragma unroll
            for (int k = 0; k < 4; ++k)         // +2 sixteen-byte units per 32-byte k-step
              wgmma_bf16_head<N_OUT, 0, 0>(d, desc_from_lo(a_t + k * 2), desc_from_lo(w_lo + k * 2), (first && k == 0) ? 0u : 1u);
          }
        }
        wg_commit();
        wg_wait<1>();                                             // the previous stage's MMAs are done: its slot is free
        if (prev >= 0) mbar_arrive(&w_empty[prev]);
        prev = (int)ws;
        first = false;
        if (++ws == (uint32_t)stages) { ws = 0; wpar ^= 1u; }
      }
    }
    wg_wait<0>();
    mbar_arrive(&w_empty[prev]);
    prev = -1;
    mbar_arrive(&a_empty[ph]);                                    // this limb's rows are no longer read -> producer
  }
  acc_fence(acc);
}

// ---- warp-specialised epilogue ---------------------------------------------------------------------------------------
// tc_conv_x3_kernel: a fourth warpgroup owns the epilogue, so the tensor pipe is not idle while an item drains.
// After an item's last MMA (phase LO), each MMA warpgroup writes its raw fp32 fragment (64 rows x 128 columns) into the
// HANDOFF, arrives on h_full and goes straight on to the next item; the epilogue warpgroup reads the handoff, arrives on
// h_empty, and applies bias / ReLU / masks / limb split / TMA stores (or, ROWS == 1, the fused pool1).
// The handoff is 128 rows of kHandRowBytes: fragment row i of MMA warpgroup cw is handoff row
// 64 cw + i (positions x channels; TR: channels x positions).  It lives in the lo-limb A buffer, whose rows are no longer
// read once phase LO is complete and which is refilled only for the next item's phase LO: the rows that do not fit there
// take a dedicated tail block.  Protocol, per item it:
//   MMA warpgroups: wait a_empty[1] phase it (BOTH warpgroups' phase-LO MMAs are complete: A_lo may be overwritten), wait
//                   h_empty phase it-1 (the tail block is drained), write, arrive h_full;
//   epilogue:       wait h_full phase it, read and work, arrive h_empty;
//   activation producer: the lo rows of item it+1 are loaded after a_empty[1] AND h_empty phase it.
// The epilogue drains the handoff early in the next item's phase HI (2/3 of the item's MMAs), so the refill of A_lo still
// lands before phase LO.
constexpr int kHandStride = 132;                   // floats per handoff row: 128 + 4 (row writes and row / column reads
constexpr int kHandRowBytes = kHandStride * 4;     // are conflict-free, as for stage_acc64's stride of 68)
constexpr int kX3EpiRegsProducer = 40, kX3EpiRegsMma = 176, kX3EpiRegsEpi = 112;
static_assert(128 * (kX3EpiRegsProducer + kX3EpiRegsEpi) + 256 * kX3EpiRegsMma <= 65536, "register file of a 512-thread CTA");

template <int N_OUT, int CB, int T>
struct ConvX3Smem {
  static constexpr int kWStageBytes = N_OUT * 128;
  // handoff rows held by the lo-limb A buffer; the rest take the tail block
  __host__ __device__ static int alo_rows(int abuf_rows) { const int r = CB * abuf_rows * 128 / kHandRowBytes; return r < 128 ? r : 128; }
  __host__ __device__ static size_t tail_bytes(int abuf_rows) { return (size_t)(128 - alo_rows(abuf_rows)) * kHandRowBytes; }
  // fixed part: alignment slack + both limbs of the A rows + TMA-store staging + handoff tail + barriers
  static size_t fixed_bytes(int abuf_rows) { return 1024 + (size_t)2 * CB * abuf_rows * 128 + kEpiStageBytes + tail_bytes(abuf_rows) + 256; }
  static int stages(int abuf_rows) {
    const long long left = 232448ll - (long long)fixed_bytes(abuf_rows);
    const int s = (int)(left / kWStageBytes);
    return s > kX3MaxStages ? kX3MaxStages : s;
  }
};

__device__ __forceinline__ float lds_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}

template <int N_OUT, int CB, int T, int FMT_A, int FMT_W, int FMT_O, int ROWS = 0>
__global__ void __launch_bounds__(512, 1)
tc_conv_x3_kernel(const __grid_constant__ CUtensorMap tmA128, const __grid_constant__ CUtensorMap tmAhh,
                  const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmOut, const ConvGeom g,
                  const int stages, const float* __restrict__ bias, const uint32_t* __restrict__ mask_bits,
                  uint32_t* __restrict__ mask_out, float* __restrict__ out_f32, const int relu, const float out_scale) {
  static_assert(FMT_A == kFmtBF16 && FMT_W == kFmtBF16, "wgmma multiplies limbs of one format");
  constexpr bool TR = N_OUT == 64;
  static_assert(!TR || T == 2, "transposed tile: one 128-position tile per MMA warpgroup");
  static_assert(TR || T == 1, "128 output channels: one tile per item (64 rows of it per MMA warpgroup)");
  static_assert(ROWS == 0 || (N_OUT == 64 && CB == 1 && T == 2), "row tiles: the 64-channel instance with two tiles");
  constexpr bool POOL = ROWS == 1;
  using S = ConvX3Smem<N_OUT, CB, T>;
  extern __shared__ uint8_t raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~(uintptr_t)1023);
  const int abuf_bytes = g.abuf_rows * 128;
  uint8_t* sA = base;                                             // [2 limbs][CB][abuf_rows][128]
  uint8_t* sW = base + (size_t)2 * CB * abuf_bytes;               // [stages][N_OUT][128]
  uint8_t* sEpi = sW + (size_t)stages * S::kWStageBytes;          // [2 warp pairs][hi, lo][32 rows][128 B]
  uint8_t* sTail = sEpi + kEpiStageBytes;                         // handoff rows [alo_rows, 128)
  const int alo_rows = S::alo_rows(g.abuf_rows);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sTail + S::tail_bytes(g.abuf_rows));
  uint64_t* a_full = bars;            // [2] per limb (0 = hi, 1 = lo)
  uint64_t* a_empty = bars + 2;       // [2]
  uint64_t* h_full = bars + 4;
  uint64_t* h_empty = bars + 5;
  uint64_t* w_full = bars + 6;        // [kX3MaxStages]
  uint64_t* w_empty = bars + 6 + kX3MaxStages;
  // shared address of handoff row r (rows past alo_rows continue in the tail block)
  const uint32_t h_alo = smem_u32(sA + (size_t)CB * abuf_bytes);
  const uint32_t h_tail = smem_u32(sTail) - (uint32_t)(alo_rows * kHandRowBytes);
  auto hrow = [&](int r) { return (r < alo_rows ? h_alo : h_tail) + (uint32_t)(r * kHandRowBytes); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], 256); }
    mbar_init(h_full, 256); mbar_init(h_empty, 128);
    for (int i = 0; i < kX3MaxStages; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], 256); }
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) prefetch_tmap(&tmW);
  if (warp == 3 && lane == 0) { prefetch_tmap(&tmA128); prefetch_tmap(&tmAhh); }
  if (warp == 12 && lane == 0) prefetch_tmap(&tmOut);
  __syncthreads();
  const int my_items = (g.num_items - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // items blockIdx.x + i*gridDim.x
  pdl_wait();                  // predecessor grid complete: global memory may be touched from here on
  pdl_trigger();

  if (warp < 4) {
    regs_dec<kX3EpiRegsProducer>();
    if (warp == 3 && lane == 0) x3_produce_acts<CB, T, ROWS>(&tmA128, &tmAhh, g, my_items, sA, a_full, a_empty, h_empty);
    else if (warp == 0 && lane == 0) x3_produce_weights<N_OUT, CB>(&tmW, my_items, stages, sW, w_full, w_empty);
  } else if (warp < 12) {
    // ===================================== MMA =====================================
    regs_inc<kX3EpiRegsMma>();
    const int cw = (warp - 4) >> 2;               // MMA warpgroup: TR: tile cw; else rows [64 cw, 64 cw + 64) of the tile
    const int tstep = ROWS ? g.Wp : 128;
    const uint32_t a_addr0 = smem_u32(sA) + (uint32_t)(TR ? cw * tstep : 64 * cw) * 128;
    const uint32_t w_lo0 = desc_lo(smem_u32(sW), 16);
    // this thread's two fragment rows in the handoff (d[4j], d[4j+1] in row r, d[4j+2], d[4j+3] in row r + 8)
    const int r0 = 64 * cw + 16 * (warp & 3) + (lane >> 2);
    const uint32_t p0 = hrow(r0) + 8 * (lane & 3), p1 = hrow(r0 + 8) + 8 * (lane & 3);
    uint32_t ws = 0, wpar = 0;
    float acc[64];
    for (int it = 0; it < my_items; ++it) {
      x3_mma_item<N_OUT, CB, T>(acc, it, g, stages, a_addr0, w_lo0, a_full, a_empty, w_full, w_empty, ws, wpar);
      mbar_wait(&a_empty[1], it & 1);             // both warpgroups are done with A_lo
      mbar_wait(h_empty, (it & 1) ^ 1);           // the previous item's handoff has been read
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(p0 + 32 * j), "f"(acc[4 * j]), "f"(acc[4 * j + 1]) : "memory");
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(p1 + 32 * j), "f"(acc[4 * j + 2]), "f"(acc[4 * j + 3]) : "memory");
      }
      mbar_arrive(h_full);
    }
  } else {
    // ===================================== epilogue =====================================
    regs_dec<kX3EpiRegsEpi>();
    // warp pair p = (warp - 12) >> 1 drains slots p, p + 2, ... (a slot = 32 positions of the item); in every slot the warp
    // of parity eg works on the 32-channel chunks 2 hf + eg, one thread per position, and the pair stores each 64-channel
    // block's hi and lo limbs through its own two 32 x 128 B staging blocks (one TMA store each).
    const int p = (warp - 12) >> 1, eg = warp & 1;
    constexpr int kSlots = POOL ? 2 : (TR ? 4 : 2);                // slots per warp pair
    constexpr int kHalves = N_OUT / 64;
    const int tstep = ROWS ? g.Wp : 128;
    // first position of slot s: TR: quarter s & 3 of tile s >> 2; else quarter s of the tile
    auto slot_q0 = [&](int q0, int s) { return TR ? q0 + (s >> 2) * tstep + (s & 3) * 32 : q0 + s * 32; };
    const int HpWp = g.Hp * g.Wp;
    uint8_t* estg_hi = sEpi + p * 8192;
    uint8_t* estg_lo = estg_hi + 4096;
    const uint32_t my_row_hi = smem_u32(estg_hi) + lane * 128, my_row_lo = smem_u32(estg_lo) + lane * 128;
    const int sw = lane & 7;
    const bool issuer = eg == 0 && lane == 0;
    auto pair_sync = [&]() { named_sync(1 + p, 64); };
    bool store_pending = false;
    for (int it = 0; it < my_items; ++it) {
      const int item = (int)blockIdx.x + it * (int)gridDim.x;
      const int q0 = x3_item_q0<T, ROWS>(g, item);
      // ReLU-backward mask words (1 bit / element), requested before the wait for the handoff
      uint32_t mbt[kSlots * kHalves];
      if (!POOL) {
#pragma unroll
        for (int k = 0; k < kSlots; ++k) {
          const int qt = slot_q0(q0, p + 2 * k) + lane;
          const bool ok = mask_bits && qt < g.Q;
#pragma unroll
          for (int hf = 0; hf < kHalves; ++hf) mbt[k * kHalves + hf] = ok ? __ldg(mask_bits + (size_t)qt * (N_OUT / 32) + hf * 2 + eg) : 0u;
        }
      }
      mbar_wait(h_full, it & 1);
      if constexpr (POOL) {
        // thread = image column x of both rows (tile 0 = row 2y, tile 1 = row 2y + 1), 32-channel chunk eg.  Scan order of the
        // 2x2 window: (row 0, x even)=0, (row 0, x odd)=1, (row 1, even)=2, (row 1, odd)=3; the first maximum wins: larger
        // value, ties to the smaller index.
        const int OH = g.H >> 1, OW = g.W >> 1;
        uint16_t* out_pool = reinterpret_cast<uint16_t*>(out_f32);             // pooled two-limb stream [B][OH+2][OW+2][hi 64 | lo 64]
        const int n = item / OH, yy = item - n * OH;
        const int c = eg;
#pragma unroll 1
        for (int k = 0; k < kSlots; ++k) {
          const int x = (p + 2 * k) * 32 + lane;
          const int px = x >> 1, odd = x & 1;
          uint16_t* prow = out_pool + (((size_t)n * (OH + 2) + yy + 1) * (OW + 2) + px + 1) * 128;
          uint32_t* crow = mask_out + (((size_t)n * OH + yy) * OW + px) * 8;
          float vs[32];
          uint32_t lower = 0u;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const float bj = __ldg(bias + c * 32 + j);
            const float a = fmaxf(lds_f32(hrow(32 * c + j) + 4 * x) + bj, 0.f), d = fmaxf(lds_f32(hrow(64 + 32 * c + j) + 4 * x) + bj, 0.f);
            vs[j] = a;
            if (d > a) { vs[j] = d; lower |= 1u << j; }
          }
          uint32_t code[4] = {0u, 0u, 0u, 0u};
          float m[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const uint32_t ks = ((lower >> j) & 1u) * 2u + (uint32_t)odd;
            const float vo = __shfl_xor_sync(0xffffffffu, vs[j], 1);
            const uint32_t ko = __shfl_xor_sync(0xffffffffu, ks, 1);
            const bool other = vo > vs[j] || (vo == vs[j] && ko < ks);
            const float mv = other ? vo : vs[j];
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
        }
      } else {
#pragma unroll 1
        for (int k = 0; k < kSlots; ++k) {
          const int s = p + 2 * k;
          const int q0w = slot_q0(q0, s);
          const int q = q0w + lane;
          const int n = q / HpWp, rem = q - n * HpWp;
          const int yp = rem / g.Wp, xp = rem - yp * g.Wp;
          const bool valid = q < g.Q && xp >= 1 && xp <= g.W && yp >= 1 && yp <= g.H;
          const size_t o_f32 = (((size_t)n * g.H + (yp - 1)) * g.W + (xp - 1)) * N_OUT;
          uint32_t mo[kHalves];
#pragma unroll
          for (int hf = 0; hf < kHalves; ++hf) {
            const int c = hf * 2 + eg;
            float v[32];
            if constexpr (TR) {
              const uint32_t col = 4 * ((s & 3) * 32 + lane);
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] = lds_f32(hrow(64 * (s >> 2) + 32 * c + j) + col);
            } else {
              lds_read32(hrow(32 * s + lane) + 128 * c, v);
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
              const uint32_t w = mbt[k * kHalves + hf];
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
            // the staging blocks may still be read by the previous TMA stores
            if (store_pending) { if (issuer) bulk_wait_read0(); pair_sync(); }
#pragma unroll
            for (int j4 = 0; j4 < 4; ++j4) {
              uint32_t hi[4], lo[4];
#pragma unroll
              for (int h = 0; h < 4; ++h) {
                const int j = 4 * j4 + h;
                if (valid) split2<FMT_O>(v[2 * j], v[2 * j + 1], hi[h], lo[h]);
                else { hi[h] = 0u; lo[h] = 0u; }                     // border / out-of-range positions store zeros
              }
              const uint32_t off = (uint32_t)(((eg * 4 + j4) ^ sw) << 4);
              asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(my_row_hi + off), "r"(hi[0]), "r"(hi[1]), "r"(hi[2]), "r"(hi[3]) : "memory");
              asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(my_row_lo + off), "r"(lo[0]), "r"(lo[1]), "r"(lo[2]), "r"(lo[3]) : "memory");
            }
            fence_proxy_async();                      // generic-proxy smem writes -> visible to the TMA engine
            pair_sync();                              // both 64-byte halves of every row are in place
            if (issuer && q0w < g.Q) {
              tma_store_2d(&tmOut, estg_hi, hf * 64, q0w);
              tma_store_2d(&tmOut, estg_lo, N_OUT + hf * 64, q0w);
              bulk_commit();
            }
            store_pending = true;
            if (out_f32 && valid) {
              float4* fp = reinterpret_cast<float4*>(out_f32 + o_f32 + c * 32);
#pragma unroll
              for (int j = 0; j < 8; ++j) fp[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
            }
          }
          if (mask_out && q < g.Q) {
#pragma unroll
            for (int hf = 0; hf < kHalves; ++hf) mask_out[(size_t)q * (N_OUT / 32) + hf * 2 + eg] = valid ? mo[hf] : 0u;
          }
        }
      }
      fence_proxy_async();                        // the handoff reads are ordered before A_lo's next TMA load
      mbar_arrive(h_empty);
    }
    if (!POOL && issuer) bulk_wait0();
    __syncwarp();
  }
}

}  // namespace tc
}  // namespace udh
