// wgmma GEMM for the fully connected head (fc1: 32768 -> 1024), bf16 operands, fp32 register accumulation.
//   D[M][N] (+)= A . B over K, tiles of 128 x 256 (two MMA warpgroups of 64 rows), k-blocks of 64, 3-stage TMA ring.
// Each operand is either K-major (contraction index contiguous in memory: tile = [rows][64 k], box (64, rows)) or
// MN-major (row/column index contiguous: tile = 64-wide column blocks of [64 k][64 mn]), which covers
//   forward   y  = x . W        A = x [B][F] K-major,      B = W [F][N] MN-major,   split-K (partials summed in split order)
//   dgrad     dx = dy . W^T     A = dy [B][N] K-major,     B = W [F][N] as [n=f][k] K-major
//   wgrad     dW = x^T . dy     A = x [B][F] MN-major,     B = dy [B][N] MN-major   (K = batch)
// with no transposed copies.  warpgroup 0: TMA producer (warp 0) | warpgroups 1-2: MMA + epilogue.
#pragma once
#include "tc_common.cuh"

namespace udh {
namespace tc {

// The contraction may run over up to three SEGMENTS: segment s reads A at (k + a_koff[s], m + a_moff[s]) and B at
// (k + b_koff[s], n + b_noff[s]).  The two-limb mode (UDH_NUMERIC_BF16X3) uses this to evaluate
// lo.hi + hi.hi + hi.lo over operands stored as [hi | lo] without duplicating anything in memory; one segment with zero
// offsets is the plain GEMM.
struct GemmGeom {
  int M, N;            // logical output size (rows beyond M / cols beyond N are not stored)
  int m_tiles, n_tiles, k_splits;
  int kb_per_split;    // k-blocks (of 64) per split, counted over all segments
  int kb_per_seg;      // k-blocks of one segment
  int a_koff[3], a_moff[3], b_koff[3], b_noff[3];
  int64_t ldc;
};

constexpr int kGemmStages = 3;
constexpr int kGemmStageBytes = 16384 + 32768;   // A 128 x 64, B 256 x 64 (bf16)

constexpr int kGemmEpiBytes = 8 * 32 * 128;      // TMA-store staging of the non-atomic epilogue: 32 rows x 32 floats per warp

// SPLIT: every split stores its partial tile in its own slab of a scratch buffer ([split][M][N]); the launcher adds the
// slabs in split order (slab_reduce), so the sum does not depend on CTA timing.  Otherwise the tile is stored through a swizzled
// shared-memory staging block and TMA (full 128-byte lines; rows / columns beyond M / N are clipped by the tensor map).
template <bool A_MN, bool B_MN, bool SPLIT, int FMT_A = kFmtBF16, int FMT_B = kFmtBF16>
__global__ void __launch_bounds__(384, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmC,
               const GemmGeom g, float* __restrict__ slab) {
  static_assert(FMT_A == kFmtBF16 && FMT_B == kFmtBF16, "wgmma multiplies operands of one format");
  extern __shared__ uint8_t raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sEpi = base + (size_t)kGemmStages * kGemmStageBytes;
  float* sStg = reinterpret_cast<float*>(sEpi + (SPLIT ? 0 : kGemmEpiBytes));   // [2 warpgroups][kStgBytes]
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sStg) + 2 * kStgBytes);
  uint64_t* full = bars;                       // [stages]
  uint64_t* empty = bars + kGemmStages;        // [stages]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kGemmStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 256); }
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) { prefetch_tmap(&tmA); prefetch_tmap(&tmB); }
  __syncthreads();
  const int num_tiles = g.m_tiles * g.n_tiles * g.k_splits;
  pdl_wait();                  // predecessor grid complete: global memory may be touched from here on
  pdl_trigger();
  const int my_tiles = (num_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  auto decode = [&](int tile, int& mt, int& nt, int& ks) {
    ks = tile % g.k_splits; tile /= g.k_splits;
    nt = tile % g.n_tiles;
    mt = tile / g.n_tiles;
  };

  if (warp < 4) {
    regs_dec<40>();
    if (warp == 0 && lane == 0) {
      uint32_t cnt = 0;
      for (int i = 0; i < my_tiles; ++i) {
        int mt, nt, ks;
        decode((int)blockIdx.x + i * (int)gridDim.x, mt, nt, ks);
        for (int kb = 0; kb < g.kb_per_split; ++kb, ++cnt) {
          const int s = cnt % kGemmStages;
          const int kg = ks * g.kb_per_split + kb;
          const int seg = kg / g.kb_per_seg;
          const int k0 = (kg - seg * g.kb_per_seg) * 64;
          const int ak = k0 + g.a_koff[seg], am = mt * 128 + g.a_moff[seg], bk = k0 + g.b_koff[seg], bn = nt * 256 + g.b_noff[seg];
          mbar_wait(&empty[s], ((cnt / kGemmStages) & 1) ^ 1);
          mbar_arrive_expect_tx(&full[s], kGemmStageBytes);
          uint8_t* sa = base + (size_t)s * kGemmStageBytes;
          uint8_t* sb = sa + 16384;
          if (A_MN) {
            for (int j = 0; j < 2; ++j) tma_load_2d(sa + j * 8192, &tmA, am + j * 64, ak, &full[s]);
          } else {
            tma_load_2d(sa, &tmA, ak, am, &full[s]);
          }
          if (B_MN) {
            for (int j = 0; j < 4; ++j) tma_load_2d(sb + j * 8192, &tmB, bn + j * 64, bk, &full[s]);
          } else {
            tma_load_2d(sb, &tmB, bk, bn, &full[s]);
          }
        }
      }
    }
  } else {
    regs_inc<232>();
    const int cw = (warp - 4) >> 2;              // MMA warpgroup: rows [64 cw, 64 cw + 64) of the tile
    const int wi = warp & 3;
    const int ew = 2 * cw + (wi & 1);            // row quarter this warp stores
    const int eg = wi >> 1;                      // 32-column chunk parity this warp stores
    const int erow = 32 * (wi & 1) + lane;
    float* stg = sStg + cw * (kStgBytes / 4);
    uint8_t* stg_tma = sEpi + (warp - 4) * 4096;  // this warp's TMA-store staging block
    const int sw = lane & 7;
    bool store_pending = false;
    uint32_t cnt = 0;
    float acc[128];
    for (int i = 0; i < my_tiles; ++i) {
      int mt, nt, ks;
      decode((int)blockIdx.x + i * (int)gridDim.x, mt, nt, ks);
      acc_fence(acc);
      int prev = -1;
      for (int kb = 0; kb < g.kb_per_split; ++kb, ++cnt) {
        const int s = cnt % kGemmStages;
        mbar_wait(&full[s], (cnt / kGemmStages) & 1);
        // this warpgroup's 64 rows: the second 64-wide column block (MN-major) or 64 rows further (K-major), 8 KB either way
        const uint32_t a_addr = smem_u32(base + (size_t)s * kGemmStageBytes) + (uint32_t)cw * 8192, b_addr = smem_u32(base + (size_t)s * kGemmStageBytes) + 16384;
        const uint32_t a_lo = desc_lo(a_addr, 16), b_lo = desc_lo(b_addr, B_MN ? 8192 : 16);
        wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_bf16<256, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, desc_from_lo(a_lo + k * (A_MN ? 128 : 2)), desc_from_lo(b_lo + k * (B_MN ? 128 : 2)),
                                                      (kb > 0 || k > 0) ? 1u : 0u);
        wg_commit();
        wg_wait<1>();
        if (prev >= 0) mbar_arrive(&empty[prev]);
        prev = s;
      }
      wg_wait<0>();
      if (prev >= 0) mbar_arrive(&empty[prev]);
      acc_fence(acc);
      const int m = mt * 128 + ew * 32 + lane;
      float* prow = slab + ((size_t)ks * g.M + m) * g.N + nt * 256;     // SPLIT: this split's partial row
#pragma unroll 1
      for (int cc = 0; cc < 4; ++cc) {
        const int c = 2 * cc + eg;
        float v[32];
        named_sync(5 + cw, 128); stage_acc64(acc, cc, stg); named_sync(5 + cw, 128);
        stg_read32(stg, erow, eg * 32, v);
        const int n0 = nt * 256 + c * 32;
        if (SPLIT) {
          if (m < g.M) {
            if (n0 + 32 <= g.N) {
#pragma unroll
              for (int j = 0; j < 8; ++j) reinterpret_cast<float4*>(prow + c * 32)[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (n0 + j < g.N) prow[c * 32 + j] = v[j];
            }
          }
        } else {
          const uint32_t my_row = smem_u32(stg_tma) + lane * 128;
          if (store_pending) { if (lane == 0) bulk_wait_read0(); __syncwarp(); }
#pragma unroll
          for (int j4 = 0; j4 < 8; ++j4)
            asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(my_row + (uint32_t)((j4 ^ sw) << 4)), "f"(v[4 * j4]), "f"(v[4 * j4 + 1]),
                         "f"(v[4 * j4 + 2]), "f"(v[4 * j4 + 3]) : "memory");
          fence_proxy_async();
          __syncwarp();
          if (lane == 0) {                          // (always commit, possibly an empty group, so the group count stays uniform)
            if (n0 < g.N && mt * 128 + ew * 32 < g.M) tma_store_2d(&tmC, stg_tma, n0, mt * 128 + ew * 32);
            bulk_commit();
          }
          store_pending = true;
        }
      }
    }
    if (!SPLIT) { if (lane == 0) bulk_wait0(); __syncwarp(); }
  }
}

// Host launcher.  C[M][N] (+)= A . B on tensor cores.  a_inner/a_outer: dims of A's tensor (innermost first); same for B.
// seg (nullable): offsets of the contraction segments (see GemmGeom), K is the length of ONE segment.
struct GemmSegments { int n; int a_koff[3], a_moff[3], b_koff[3], b_noff[3]; };

template <bool A_MN, bool B_MN, bool SPLIT, int FMT_A = kFmtBF16, int FMT_B = kFmtBF16>
inline int launch_gemm(const void* A, uint64_t a_inner, uint64_t a_outer, const void* Bm, uint64_t b_inner, uint64_t b_outer,
                       float* C, int64_t ldc, int M, int N, int K, int k_splits, const GemmSegments* seg, cudaStream_t st) {
  GemmGeom g;
  g.M = M; g.N = N; g.ldc = ldc;
  g.m_tiles = (M + 127) / 128; g.n_tiles = (N + 255) / 256;
  const int nseg = seg ? seg->n : 1;
  g.kb_per_seg = (K + 63) / 64;
  const int kb = g.kb_per_seg * nseg;
  g.k_splits = k_splits;
  g.kb_per_split = (kb + k_splits - 1) / k_splits;
  UDH_REQUIRE(g.kb_per_split * k_splits == kb, "tc gemm: k-blocks (%d) must divide evenly into %d splits", kb, k_splits);
  for (int i = 0; i < 3; ++i) {
    g.a_koff[i] = seg && i < nseg ? seg->a_koff[i] : 0; g.a_moff[i] = seg && i < nseg ? seg->a_moff[i] : 0;
    g.b_koff[i] = seg && i < nseg ? seg->b_koff[i] : 0; g.b_noff[i] = seg && i < nseg ? seg->b_noff[i] : 0;
  }
  CUtensorMap tmA, tmB;
  uint64_t dA[2] = {a_inner, a_outer}, sA[2] = {2, a_inner * 2};
  uint32_t boxA[2] = {64, A_MN ? 64u : 128u};
  int rc = make_tmap_bf16(&tmA, A, 2, dA, sA, boxA);
  if (rc != UDH_OK) return rc;
  uint64_t dB[2] = {b_inner, b_outer}, sB[2] = {2, b_inner * 2};
  uint32_t boxB[2] = {64, B_MN ? 64u : 256u};
  rc = make_tmap_bf16(&tmB, Bm, 2, dB, sB, boxB);
  if (rc != UDH_OK) return rc;
  // output map for the TMA-store epilogue: fp32 [M][ldc], box = 32 floats (128 B) x 32 rows
  CUtensorMap tmC;
  uint64_t dC[2] = {(uint64_t)N, (uint64_t)M}, sC[2] = {4, (uint64_t)ldc * 4};
  uint32_t boxC[2] = {32, 32};
  rc = make_tmap(&tmC, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, C, 2, dC, sC, boxC);
  if (rc != UDH_OK) return rc;
  const size_t smem = 1024 + (size_t)kGemmStages * kGemmStageBytes + (SPLIT ? 0 : kGemmEpiBytes) + 2 * kStgBytes + 256;
  auto kern = tc_gemm_kernel<A_MN, B_MN, SPLIT, FMT_A, FMT_B>;
  UDH_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int sms = persistent_ctas();
  const int tiles = g.m_tiles * g.n_tiles * g.k_splits;
  float* slab = nullptr;
  if (SPLIT) {
    UDH_REQUIRE(ldc == N, "tc gemm: split-K needs a dense output (ldc %lld, N %d)", (long long)ldc, N);
    slab = slab_scratch((size_t)k_splits * M * N, st);
    if (!slab) return UDH_ECUDA;
  }
  launch_chain(kern, dim3(tiles < sms ? tiles : sms), dim3(384), smem, st, tmA, tmB, tmC, g, slab);
  if (int rc2 = check_launch("tc_gemm_kernel")) return rc2;
  if (!SPLIT) return UDH_OK;
  SlabSegments t;
  t.count = 1;
  t.s[0] = SlabSegment{slab, C, (size_t)M * N, k_splits, M * N};
  return slab_reduce(t, st);
}

}  // namespace tc
}  // namespace udh
