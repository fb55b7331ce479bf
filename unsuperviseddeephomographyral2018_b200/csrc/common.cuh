// Shared helpers of libudh (error reporting, launch checks, warp/block reductions).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <stdlib.h>

#include "../../include/udh.h"

namespace udh {

void set_error(const char* fmt, ...);

// ---- in-library instrumentation (bench.py reads it): kernel-launch counter and per-phase CUDA-event timers ----
enum ProfTag {
  PROF_CONV_FWD0 = 0,    // +layer (0..7)
  PROF_CONV_DGRAD0 = 8,  // +layer
  PROF_CONV_WGRAD0 = 16, // +layer
  PROF_POOL_FWD = 24, PROF_POOL_BWD, PROF_FC_FWD, PROF_FC_BWD, PROF_DLT, PROF_WARP_FWD, PROF_WARP_BWD, PROF_SSIM,
  PROF_H4P_LOSS, PROF_ADAM, PROF_ELTWISE, PROF_TC_PREP,
  PROF_MB_BASE, PROF_MB_DOWN, PROF_MB_ACC, PROF_MB_COLLAPSE,   // the mosaic's multi-band blend, by phase
  PROF_NUM_TAGS
};
extern unsigned long long g_launches;
extern int g_sm_reserve;      // SMs the persistent tensor-core kernels leave free (udh_set_sm_reserve)
extern int g_sm_reserve_top;  // SMs the conv4_x backward kernels leave free (udh_set_sm_reserve_top): these few launches run
                              // while the fc-gradient allreduce occupies SMs; they have <= 2 items per CTA either way
// SMs of the H100 SXM: sizes the grids of the grid-stride (non-persistent) kernels
constexpr int kSmCount = 132;
// CTAs a persistent one-CTA-per-SM kernel should launch on the current device
inline int persistent_ctas() {
  int dev = 0, sms = kSmCount;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int n = sms - g_sm_reserve;
  return n > 0 ? n : 1;
}
extern int g_bwd_marker_layer, g_sm_reserve_marker;   // udh_set_bwd_marker / udh_set_sm_reserve_marker
// SMs the persistent backward kernels of conv layer i leave free: the global reserve, conv4_x's (udh_set_sm_reserve_top), and
// from the marker layer down the SMs handed to the second stream's kernel (udh_set_sm_reserve_marker)
inline int bwd_sm_reserve(int i, int reserve_all) {
  int r = (i >= 6 && g_sm_reserve_top > reserve_all) ? g_sm_reserve_top : reserve_all;
  if (g_bwd_marker_layer >= 0 && i <= g_bwd_marker_layer && g_sm_reserve_marker > r) r = g_sm_reserve_marker;
  return r;
}
int bwd_marker_record(int layer, cudaStream_t st);   // udh_set_bwd_marker: event before layer's backward kernels
void prof_begin(int tag, cudaStream_t st);
void prof_end(int tag, cudaStream_t st);
struct ProfScope {
  int tag; cudaStream_t st;
  ProfScope(int t, cudaStream_t s) : tag(t), st(s) { prof_begin(tag, st); }
  ~ProfScope() { prof_end(tag, st); }
};

// ---- split reductions with a result that does not depend on CTA timing ----
// Floating-point addition does not associate, so CTAs adding partial results of the same outputs with atomics give a
// result that changes from run to run (and Adam amplifies the difference over the steps).  Such CTAs instead store their
// partials in their own slab of a scratch buffer, and slab_reduce adds the slabs to the outputs in slab order.
struct SlabSegment { const float* slab; float* dst; size_t stride; int nslab; int n; };   // dst[e] += sum_k slab[k*stride + e]
struct SlabSegments { int count; SlabSegment s[16]; };
float* slab_scratch(size_t floats, cudaStream_t st);   // grow-only buffer of the current device; nullptr (+ error) on failure
int slab_reduce(const SlabSegments& segs, cudaStream_t st);

inline int check_launch(const char* what) {
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return UDH_ECUDA;
  }
  return UDH_OK;
}

#define UDH_REQUIRE(cond, ...)        \
  do {                                \
    if (!(cond)) {                    \
      udh::set_error(__VA_ARGS__);    \
      return UDH_EINVAL;              \
    }                                 \
  } while (0)

#define UDH_CUDA(call)                                                      \
  do {                                                                      \
    cudaError_t e__ = (call);                                               \
    if (e__ != cudaSuccess) {                                               \
      udh::set_error("%s failed: %s", #call, cudaGetErrorString(e__));      \
      return UDH_ECUDA;                                                     \
    }                                                                       \
  } while (0)

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// ---- programmatic dependent launch (PDL) for the back-to-back kernels of the bf16 step ---------------------------------
// A kernel launched through launch_chain() may be scheduled while its predecessor in the stream is still draining: its CTAs
// take over SMs as the predecessor's CTAs exit and run their prologue (barrier init, tensor-map prefetch)
// early.  Every such kernel calls pdl_wait() before its first global-memory access (it returns once the predecessor grid
// has completed and its writes are visible) and pdl_trigger() right after, so completion is transitive along the chain.
// UDH_PDL=0 in the environment falls back to plain launches (griddepcontrol.wait is then a no-op).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
inline bool pdl_enabled() {
  static int on = -1;
  if (on < 0) { const char* e = getenv("UDH_PDL"); on = (e && e[0] == '0') ? 0 : 1; }
  return on != 0;
}
template <typename... KArgs, typename... Args>
inline void launch_chain(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = pdl_enabled() ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);     // errors surface through check_launch()
}

// ---- the uint8 image the reference hands to cv2 ------------------------------------------------------------------------
// denorm_img(normalised augmented image).astype(uint8) of one uint8 value x of channel c (utils/utils.py:406-413), with
// a = the image's 5 augmentation parameters of udh_prep_inputs_u8_ex (gamma, brightness, 3 colour gains) or null.
// gamma: pow in fp64 rounded once to fp32 (a correctly rounded powf, reproducible on the host); the rest is the fp32
// arithmetic of udh_prep_inputs_u8_ex.  denorm_img multiplies the fp32 value by a float64 std and adds a float64 mean in
// two roundings (no FMA), and astype(uint8) truncates.  Callers tabulate it per (sample, image, channel).
__device__ __forceinline__ uint8_t denorm_u8(int x, int c, const float* a) {
  const float mean = c == 0 ? 118.93f : (c == 1 ? 113.97f : 102.60f);
  const float sd = c == 0 ? 69.85f : (c == 1 ? 68.81f : 72.45f);
  const double mean64 = c == 0 ? 118.93 : (c == 1 ? 113.97 : 102.60);    // float64 numpy arrays
  const double sd64 = c == 0 ? 69.85 : (c == 1 ? 68.81 : 72.45);
  float v = (float)x;
  if (a) {
    v = (float)pow((double)v, (double)a[0]);
    v = __fmul_rn(v, a[1]);
    v = __fmul_rn(v, a[2 + c]);
    v = fminf(fmaxf(v, 0.0f), 255.0f);
  }
  const float n = __fdiv_rn(__fsub_rn(v, mean), sd);
  const double d = __dadd_rn(__dmul_rn((double)n, sd64), mean64);
  const int t = (int)d;                                                  // truncation toward zero
  return (uint8_t)(t < 0 ? 0 : (t > 255 ? 255 : t));
}

// OpenCV's BORDER_REFLECT_101 (gfedcb|abcdefgh|gfedcba): the index in [0, n) that i reads, for any n >= 2 and any i.  The
// pattern has period 2n - 2, so |i| is folded into one period and its upper half mirrored; reflecting once is not enough
// when the reach exceeds n - 1 (a 5-tap filter on a side of 2).
__host__ __device__ __forceinline__ int reflect101(int i, int n) {
  if (i >= 0 && i < n) return i;
  const int p = 2 * n - 2;
  const int r = (i < 0 ? -i : i) % p;
  return r < n ? r : p - r;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum of NV values per thread; result valid in thread 0.  `scratch` holds NV * 32 elements of T.
template <typename T, int NV>
__device__ __forceinline__ void block_sum(T (&v)[NV], T* scratch) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = warp_sum(v[i]);
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) scratch[i * 32 + warp] = v[i];
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      T x = lane < nwarp ? scratch[i * 32 + lane] : T(0);
      v[i] = warp_sum(x);
    }
  }
}

}  // namespace udh
