// Carve-up of the tensor-core region of the regressor workspace, shared by the single-pass bf16 mode (conv_tc.cu) and the
// error-compensated two-limb mode (conv_x3.cu).  `limbs` = 1: one bf16 value per element; `limbs` = 2: every stream row
// holds [hi(C) | lo(C)] 16-bit channels (the value is hi + lo), packed weights hold a hi and a lo block per k-block.
#pragma once
#include "common.cuh"

namespace udh {
namespace tcl {

struct ConvSpec { int cin, cout, div; };
static const ConvSpec kConv[8] = {{2, 64, 1}, {64, 64, 1}, {64, 64, 2}, {64, 64, 2}, {64, 128, 4}, {128, 128, 4}, {128, 128, 8}, {128, 128, 8}};

inline size_t al256(size_t n) { return (n + 255) / 256 * 256; }
inline unsigned grid1d(size_t want, size_t cap) { return (unsigned)(want < cap ? (want ? want : 1) : cap); }

// byte offsets inside the tensor-core region of the workspace
struct TcLayout {
  size_t P[11];      // padded 16-bit activations: 0..7 conv outputs, 8..10 pool outputs
  size_t G[11];      // padded 16-bit gradients w.r.t. the same tensors (pre-activation for convs)
  size_t numel[11];  // padded element counts (logical channels)
  size_t wf[8], wd[8];   // packed 16-bit weights, forward / dgrad (rotated)
  size_t Mb[8];      // 1-bit ReLU masks [Q][C/32] uint32 of the conv outputs a dgrad needs (layers 0, 2, 4, 6)
  size_t Px[3];      // max-pool routing codes [B][H/2][W/2][C/8] uint32 (3 bits per channel), written by the forward
  size_t fc_x, fc_w, fc_dy;   // 16-bit copies for the fc1 GEMMs: x [B,F], W [F,1024], dy [B,1024] (x limbs)
  size_t fc_end;     // end of the fc1 copies: they come first, so fc1 alone runs in a region of fc_end bytes (udh_debug_fc1)
  size_t total;
  int limbs;
  TcLayout(int B, int P_, int limbs_ = 1) : limbs(limbs_) {
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o += al256(bytes); return r; };
    const size_t eb = 2 * (size_t)limbs;                         // bytes per logical element
    const size_t feat = (size_t)(P_ / 8) * (P_ / 8) * 128;
    fc_x = take((size_t)B * feat * eb);
    fc_w = take(feat * 1024 * eb);
    fc_dy = take((size_t)B * 1024 * eb);
    fc_end = o;
    for (int i = 0; i < 8; ++i) {
      const size_t s = P_ / kConv[i].div + 2;
      numel[i] = (size_t)B * s * s * kConv[i].cout;
    }
    numel[8] = (size_t)B * (P_ / 2 + 2) * (P_ / 2 + 2) * 64;
    numel[9] = (size_t)B * (P_ / 4 + 2) * (P_ / 4 + 2) * 64;
    numel[10] = (size_t)B * (P_ / 8 + 2) * (P_ / 8 + 2) * 128;
    for (int i = 0; i < 11; ++i) P[i] = take(numel[i] * eb);
    for (int i = 0; i < 11; ++i) G[i] = take(numel[i] * eb);
    for (int i = 0; i < 8; ++i) { wf[i] = take((size_t)9 * kConv[i].cin * kConv[i].cout * eb); wd[i] = take((size_t)9 * kConv[i].cin * kConv[i].cout * eb); }
    for (int i = 0; i < 8; ++i) Mb[i] = (i % 2 == 0) ? take(numel[i] / 8) : 0;
    for (int i = 0; i < 3; ++i) Px[i] = take((size_t)B * (P_ >> (i + 1)) * (P_ >> (i + 1)) * (i == 2 ? 16 : 8) * 4);
    total = o;
  }
};

template <typename T>
inline T* at(void* ws, size_t off) { return reinterpret_cast<T*>(reinterpret_cast<char*>(ws) + off); }

// input tensor index (into P / G) of conv layer i (i >= 1)
inline int input_of(int i) { return (i == 2 || i == 4 || i == 6) ? 8 + (i - 2) / 2 : i - 1; }

}  // namespace tcl
}  // namespace udh

#define UDH_TRY(call)                \
  do {                               \
    int rc__ = (call);               \
    if (rc__ != UDH_OK) return rc__; \
  } while (0)
