// wgmma / TMA tensor-core path of the regressor's convolutions (UDH_NUMERIC_BF16).
#pragma once
#include "common.cuh"

namespace udh {

// extra workspace the tensor-core path needs behind the fp32 carve-up (bf16 activations, packed weights, ...)
size_t tc_workspace_bytes(int B, int P, int numeric_mode);

// zero the padded streams once after the workspace is allocated (their borders are never written afterwards)
int tc_workspace_init(void* ws, size_t tc_off, int B, int P, cudaStream_t st);

// conv1_1 .. conv4_2 + the three max-pools; writes the fp32 activations the rest of the pipeline reads
// (act_off[7]: conv4_2 output) and keeps bf16 copies for the backward.
int tc_cnn_fwd_convs(const float* params, const size_t* param_off, const float* I1, const float* I2, void* ws,
                     const size_t* act_off, size_t tc_off, int B, int P, cudaStream_t st);

// backward of the conv stack given gA = d(pre-activation of conv4_2) [B,P/8,P/8,128] fp32.
int tc_cnn_bwd_convs(const float* params, const size_t* param_off, const float* I1, const float* I2, float* grads, float* gA,
                     float* gB, void* ws, const size_t* act_off, size_t tc_off, int B, int P, cudaStream_t st);

// fc1 (32768 -> 1024) on tensor cores; bf16 copies of x / W / dy live in the tensor-core workspace region.
int tc_fc1_fwd(const float* x, const float* w, float* acc, void* ws, size_t tc_off, int B, int P, bool w_mirror_current, cudaStream_t st);
void* tc_fc1_mirror(void* ws, size_t tc_off, int B, int P);
int tc_fc1_bwd(const float* dy, float* dW, float* dx, void* ws, size_t tc_off, int B, int P, cudaStream_t st);
// bytes at the start of the tensor-core region that fc1's forward / backward touch (limbs = 1: bf16 mode, 2: two-limb mode)
size_t fc1_region_bytes(int B, int P, int limbs);

// ---- UDH_NUMERIC_BF16X3 (conv_x3.cu): the same pipeline on two-limb streams, lo.hi + hi.hi + hi.lo per product ----------
size_t x3_workspace_bytes(int B, int P);
int x3_workspace_init(void* ws, size_t tc_off, int B, int P, cudaStream_t st);
int x3_cnn_fwd_convs(const float* params, const size_t* param_off, const float* I1, const float* I2, void* ws,
                     const size_t* act_off, size_t tc_off, int B, int P, cudaStream_t st);
int x3_cnn_bwd_convs(const float* params, const size_t* param_off, const float* I1, const float* I2, float* grads, float* gA,
                     void* ws, size_t tc_off, int B, int P, cudaStream_t st);
int x3_fc1_fwd(const float* x, const float* w, float* acc, void* ws, size_t tc_off, int B, int P, bool w_mirror_current, cudaStream_t st);
void* x3_fc1_mirror(void* ws, size_t tc_off, int B, int P);
int x3_materialize_acts(void* ws, const size_t* act_off, size_t tc_off, int B, int P, cudaStream_t st);
int x3_fc1_bwd(const float* dy, float* dW, float* dx, void* ws, size_t tc_off, int B, int P, cudaStream_t st);

// udh_debug_tc_pool: the step's 2x2 max-pool kernels of each tensor-core mode on fp32 tensors, through zeroed streams
// s_in (shaped like in) and s_out (shaped like out) of that mode's format
int tc_debug_pool(const float* in, float* out, uint32_t* codes, const float* dout, float* din, uint16_t* s_in, uint16_t* s_out, int B,
                  int H, int W, int C, cudaStream_t st);
int x3_debug_pool(const float* in, float* out, uint32_t* codes, const float* dout, float* din, uint16_t* s_in, uint16_t* s_out, int B,
                  int H, int W, int C, cudaStream_t st);

}  // namespace udh
