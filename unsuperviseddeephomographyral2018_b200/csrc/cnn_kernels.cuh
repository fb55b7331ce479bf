// Launchers of the regressor's building blocks (Row C).  fp32 CUDA-core kernels live in cnn_simt.cu; the
// wgmma tensor-core path lives in conv_tc.cu.  All tensors NHWC fp32 unless noted.
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace udh {

// out[n,y,x,co] = act( sum_{ky,kx,ci} in[n,y+ky-1,x+kx-1,ci] * w[ky,kx,ci,co] + bias[co] ), zero padding.
// `in1` != nullptr: the input is two single-channel planes (Cin == 2: I1 -> channel 0, I2 -> channel 1).
// relu: apply max(.,0).  mask_src != nullptr: multiply the result by [mask_src > 0] (ReLU backward of the layer
// whose forward output is mask_src — used when this kernel runs as a dgrad).
int conv3x3_simt(const float* in0, const float* in1, const float* w, const float* bias, const float* mask_src,
                 float* out, int B, int H, int W, int Cin, int Cout, int relu, cudaStream_t st);

// dW[ky,kx,ci,co] += sum_{n,y,x} x[n,y+ky-1,x+kx-1,ci] * g[n,y,x,co];  db[co] += sum g   (atomic accumulation)
int wgrad3x3_simt(const float* x0, const float* x1, const float* g, float* dW, float* db, int B, int H, int W,
                  int Cin, int Cout, cudaStream_t st);
// How wgrad3x3_simt splits the B (H/8) (W/16) pixel tiles: CTA x walks tiles [x tiles_per_cta, (x+1) tiles_per_cta) and
// each of its threads sums the rows r = s, s + row_split, ... of every tile; every such partial is one atomicAdd.
struct WgradPartition { int ctas_x, tiles_per_cta, row_split; };
WgradPartition wgrad3x3_partition(int B, int H, int W, int Cin, int Cout, bool two_plane);

// wrot[ky,kx,co,ci] = w[2-ky,2-kx,ci,co]  (weights of the dgrad convolution)
int rotate_weights(const float* w, float* wrot, int Cin, int Cout, cudaStream_t st);

int maxpool2x2_fwd(const float* in, float* out, int B, int H, int W, int C, cudaStream_t st);
// din[p] = dout[pool(p)] if p is the (first) arg-max of its window and in[p] > 0 (ReLU mask of the producer), else 0
int maxpool2x2_bwd(const float* in, const float* dout, float* din, int B, int H, int W, int C, cudaStream_t st);

// C[M,N] (+)= op(A)[M,K] . op(B)[K,N] with explicit element strides; split_k > 1 accumulates atomically into a
// zero-initialised (or to-be-accumulated) C.  accumulate != 0 -> C += (always atomic-add semantics).
int sgemm_simt(const float* A, int64_t a_rs, int64_t a_cs, const float* Bm, int64_t b_rs, int64_t b_cs, float* C,
               int64_t ldc, int M, int N, int K, int split_k, int accumulate, cudaStream_t st);

// fc1 of UDH_NUMERIC_FP32 (F -> 1024): acc[B,1024] (zeroed by the caller) += x[B,F] . W[F,1024];
// backward dW[F,1024] += x^T . dy, dx[B,F] = dy . W^T
int fc1_fwd_simt(const float* x, const float* w, float* acc, int B, int F, cudaStream_t st);
int fc1_bwd_simt(const float* x, const float* w, const float* dy, float* dW, float* dx, int B, int F, cudaStream_t st);

// y = relu(x + bias) -> act (nullable) ; drop = act * keep * 2 (if mask != nullptr, mask generated from seed/salt)
int bias_act_dropout(const float* x, const float* bias, float* act, float* drop, uint8_t* mask, int rows, int cols,
                     int relu, int gen_mask, uint64_t seed, uint64_t salt, cudaStream_t st);
// drop = x * keep * 2, mask generated (rows*cols elements)
int dropout_fwd(const float* x, float* drop, uint8_t* mask, size_t n, uint64_t seed, uint64_t salt, cudaStream_t st);
// g *= (mask ? 2*mask : 1) * [act > 0]
int drop_relu_bwd(float* g, const uint8_t* mask, const float* act, size_t n, cudaStream_t st);
// db[c] += sum_r g[r,c]
int colsum_accum(const float* g, float* db, int rows, int cols, cudaStream_t st);

}  // namespace udh
