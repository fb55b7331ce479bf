// sm_90a building blocks written as inline PTX: mbarrier, TMA (cp.async.bulk.tensor), wgmma with shared-memory matrix
// descriptors, register reallocation.  No CUTLASS/CuTe dependency.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace udh {
namespace tc {

// ------------------------------------------------------------------------------------------------ host: tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled through the runtime's driver entry point (libudh does not link libcuda, so the library
// still loads on a box without a driver — needed by the CPU-side ABI tests).
inline EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// `rank` dims (innermost first), 128-byte swizzle, zero fill out of bounds.  The inner box extent must span 128 bytes.
inline int make_tmap(CUtensorMap* map, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled is unavailable (no CUDA driver?)"); return UDH_ECUDA; }
  cuuint64_t gdim[5], gstr[5];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i + 1];   // stride of dim i+1 (dim 0 is contiguous)
  CUresult r = fn(map, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return UDH_ECUDA; }
  return UDH_OK;
}

inline int make_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                          const uint32_t* box) {
  return make_tmap(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, rank, dims, strides_bytes, box);
}

// ------------------------------------------------------------------------------------------------ device: PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile("{\n\t.reg .pred P1;\n\telect.sync _|P1, 0xffffffff;\n\tselp.u32 %0, 1, 0, P1;\n\t}" : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// Bounded wait: a protocol bug traps after ~2 s (launch error) instead of hanging the GPU.
// No printf here: any call in a kernel makes ptxas serialise every wgmma of it (C7510).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = globaltimer_ns();
  while (!mbar_try_wait(bar, parity)) {
    if (globaltimer_ns() - t0 > 2000000000ull) asm volatile("trap;");
  }
}

__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, int c0, int c1, int c2, int c3, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}

// TMA store smem -> global (bulk async group), 2D tile
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }


// ---- descriptors -------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, 128-byte swizzle.  start: smem byte address; lbo/sbo in bytes;
// base_offset = (start >> 7) & 7 when the start is not on a 1024-byte swizzle-pattern boundary.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t start, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t base_offset) {
  uint64_t d = 0;
  d |= (uint64_t)((start & 0x3FFFFu) >> 4);             // [0,14)  start address >> 4
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;    // [16,30) leading byte offset >> 4
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;    // [32,46) stride byte offset >> 4
  d |= (uint64_t)(base_offset & 7u) << 49;              // [49,52) matrix base offset
  d |= (uint64_t)1 << 62;                               // [62,64) layout type: SWIZZLE_128B
  return d;
}

// Fast path for issue loops: the upper word is constant (SBO = 1024 B, SWIZZLE_128B, base_offset 0); the lower
// word is (start >> 4) | (LBO >> 4) << 16, so stepping the start address is one 32-bit add.
constexpr uint32_t kDescHiSw128 = (1024u >> 4) | (1u << 30);
__device__ __forceinline__ uint32_t desc_lo(uint32_t start, uint32_t lbo_bytes) { return ((start & 0x3FFFFu) >> 4) | ((lbo_bytes >> 4) << 16); }
__device__ __forceinline__ uint64_t desc_from_lo(uint32_t lo) { return ((uint64_t)kDescHiSw128 << 32) | lo; }

constexpr int kFmtF16 = 0, kFmtBF16 = 1;   // 16-bit limb formats

// ---- two-limb split of fp32 values (UDH_NUMERIC_BF16X3) ------------------------------------------------------------
// x = hi + lo with hi = round16(x), lo = round16(x - hi) (x - hi is exact in fp32).  The product of two split values is
// evaluated on the tensor pipe as hi*hi + hi*lo + lo*hi with fp32 accumulation; the dropped lo*lo term and the residual
// of the split are both <= 2^-16 |x y| for bf16 limbs (2^-22 for fp16 limbs).  Two values are packed per 32-bit word.
template <int FMT>
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  if (FMT == kFmtBF16) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    const __nv_bfloat162 l = __floats2bfloat162_rn(a - __low2float(h), b - __high2float(h));
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
  } else {
    const __half2 h = __floats2half2_rn(a, b);
    const __half2 l = __floats2half2_rn(a - __low2float(h), b - __high2float(h));
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
  }
}
// value of a packed pair of limbs: (hi.x + lo.x, hi.y + lo.y)
template <int FMT>
__device__ __forceinline__ float2 join2(uint32_t hi, uint32_t lo) {
  if (FMT == kFmtBF16) {
    const __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(&hi), l = *reinterpret_cast<const __nv_bfloat162*>(&lo);
    return make_float2(__low2float(h) + __low2float(l), __high2float(h) + __high2float(l));
  } else {
    const __half2 h = *reinterpret_cast<const __half2*>(&hi), l = *reinterpret_cast<const __half2*>(&lo);
    return make_float2(__low2float(h) + __low2float(l), __high2float(h) + __high2float(l));
  }
}

// ---- wgmma: one warpgroup computes D[64 x N] (+)= A[64 x 16] . B[16 x N], bf16 operands from shared-memory descriptors,
// fp32 accumulators in registers.  TA / TB: 1 = MN-major operand.  Fragment of thread (warp w of the warpgroup, lane l):
// d[i] = D[16 w + l/4 + 8 ((i >> 1) & 1)][8 (i >> 2) + 2 (l % 4) + (i & 1)].
template <int N> struct Wgmma;
template <> struct Wgmma<64> {
  template <int TA, int TB>
  static __device__ __forceinline__ void run(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
                 "}, %32, %33, p, 1, 1, %35, %36;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
};
template <> struct Wgmma<128> {
  template <int TA, int TB>
  static __device__ __forceinline__ void run(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
                 "}, %64, %65, p, 1, 1, %67, %68;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
};
template <> struct Wgmma<192> {
  template <int TA, int TB>
  static __device__ __forceinline__ void run(float (&d)[96], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n192k16.f32.bf16.bf16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
                 "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
                 "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
                 "}, %96, %97, p, 1, 1, %99, %100;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
                   "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
                   "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
                   "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
                   "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
                 : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
};
template <> struct Wgmma<256> {
  template <int TA, int TB>
  static __device__ __forceinline__ void run(float (&d)[128], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
                 "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
                 "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
                 "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
                 "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
                 "}, %128, %129, p, 1, 1, %131, %132;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
                   "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
                   "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
                   "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
                   "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
                   "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
                   "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
                   "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
                   "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
                 : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
};

template <int N, int TA, int TB, int K>
__device__ __forceinline__ void wgmma_bf16(float (&d)[K], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  static_assert(K == N / 2, "accumulator fragment size");
  Wgmma<N>::template run<TA, TB>(d, adesc, bdesc, accumulate);
}
// the first N/2 registers of a wider fragment (its first N columns)
template <int N, int TA, int TB, int K>
__device__ __forceinline__ void wgmma_bf16_head(float (&d)[K], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  static_assert(K >= N / 2, "accumulator fragment size");
  Wgmma<N>::template run<TA, TB>(*reinterpret_cast<float(*)[N / 2]>(&d[0]), adesc, bdesc, accumulate);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int K> __device__ __forceinline__ void acc_fence(float (&d)[K]) {
#pragma unroll
  for (int i = 0; i < K; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int K> __device__ __forceinline__ void acc_zero(float (&d)[K]) {
#pragma unroll
  for (int i = 0; i < K; ++i) d[i] = 0.f;
}

// register budget moves between the producer warpgroup and the MMA warpgroups
template <int R> __device__ __forceinline__ void regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
__device__ __forceinline__ void named_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// ---- accumulator rows as "one thread = one row" ------------------------------------------------------------------------
// The epilogues work on 32 consecutive columns of one accumulator row per thread.  A warpgroup writes 64 columns of its
// 64-row fragment into a [64][kStgStride] fp32 block (stage_acc64), meets at a named barrier, and every thread then reads
// 32 columns of one row (stg_read32).  The stride of 68 floats keeps both the fragment writes and the row reads
// bank-conflict free.
constexpr int kStgStride = 68;
constexpr int kStgBytes = 64 * kStgStride * 4;
// columns [64 blk, 64 blk + 64) of the fragment d (blk may be a runtime value: every register index stays static)
template <int K>
__device__ __forceinline__ void stage_acc64(const float (&d)[K], int blk, float* stg) {
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  float* r0 = stg + (16 * w + (lane >> 2)) * kStgStride + 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < K / 4; ++j) {
    if ((j >> 3) != blk) continue;
    const int c = 8 * (j & 7);
    *reinterpret_cast<float2*>(r0 + c) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(r0 + 8 * kStgStride + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
// every (row, column pair) of this warpgroup's 64-row fragment d to off(row, column) (nullptr: not stored); column is even
template <int K, typename Off>
__device__ __forceinline__ void store_acc(const float (&d)[K], Off off) {
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const int r = 16 * w + (lane >> 2);
#pragma unroll
  for (int j = 0; j < K / 4; ++j) {
    const int c = 8 * j + 2 * (lane & 3);
    if (float* p = off(r, c)) *reinterpret_cast<float2*>(p) = make_float2(d[4 * j], d[4 * j + 1]);
    if (float* p = off(r + 8, c)) *reinterpret_cast<float2*>(p) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
// v[j] = staged[row][c0 + j]
__device__ __forceinline__ void stg_read32(const float* stg, int row, int c0, float (&v)[32]) {
  const float4* p = reinterpret_cast<const float4*>(stg + row * kStgStride + c0);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 x = p[j];
    v[4 * j] = x.x; v[4 * j + 1] = x.y; v[4 * j + 2] = x.z; v[4 * j + 3] = x.w;
  }
}

}  // namespace tc
}  // namespace udh
