// Orchestration of the 4-point regressor (Row C): workspace layout, forward and backward schedules.
// Reference: code/homography_model.py:88-133 (_conv2d/_conv_block/_maxpool2d/_vgg) and the TF autodiff of it
// (opt_step.compute_gradients, code/homography_CNN_synthetic.py:258-269).
#include "cnn_kernels.cuh"
#include "conv_tc.cuh"

namespace udh {

namespace {

struct ConvSpec { int cin, cout, div; };   // div: spatial size = P / div
const ConvSpec kConv[8] = {{2, 64, 1}, {64, 64, 1}, {64, 64, 2}, {64, 64, 2}, {64, 128, 4}, {128, 128, 4}, {128, 128, 8}, {128, 128, 8}};

inline size_t round32(size_t n) { return (n + 31) / 32 * 32; }

struct ParamLayout {
  size_t off[20], numel[20], total;
  explicit ParamLayout(int P) {
    size_t o = 0;
    int t = 0;
    for (int i = 0; i < 8; ++i) {
      numel[t] = (size_t)9 * kConv[i].cin * kConv[i].cout; off[t] = o; o += round32(numel[t]); ++t;
      numel[t] = kConv[i].cout; off[t] = o; o += round32(numel[t]); ++t;
    }
    const size_t feat = (size_t)(P / 8) * (P / 8) * 128;
    numel[t] = feat * 1024; off[t] = o; o += round32(numel[t]); ++t;
    numel[t] = 1024; off[t] = o; o += round32(numel[t]); ++t;
    numel[t] = 1024 * 8; off[t] = o; o += round32(numel[t]); ++t;
    numel[t] = 8; off[t] = o; o += round32(numel[t]); ++t;
    total = o;
  }
};

// Workspace carve-up (byte offsets, 256-byte aligned).
struct Workspace {
  size_t act[12];      // 0..7 conv outputs, 8..10 pool outputs, 11 fc1 (post-ReLU)
  size_t act_numel[12];
  size_t a4d, fc1_acc, fc1d, dfc1, gA, gB, wrot, mask1, mask2, tc;
  size_t total;
  int B, P;
  Workspace(int B_, int P_, int numeric_mode) : B(B_), P(P_) {
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 255) / 256 * 256; return r; };
    for (int i = 0; i < 8; ++i) {
      const size_t s = P / kConv[i].div;
      act_numel[i] = (size_t)B * s * s * kConv[i].cout;
    }
    act_numel[8] = (size_t)B * (P / 2) * (P / 2) * 64;
    act_numel[9] = (size_t)B * (P / 4) * (P / 4) * 64;
    act_numel[10] = (size_t)B * (P / 8) * (P / 8) * 128;
    act_numel[11] = (size_t)B * 1024;
    for (int i = 0; i < 12; ++i) act[i] = take(act_numel[i] * 4);
    const size_t feat = (size_t)(P / 8) * (P / 8) * 128;
    a4d = take((size_t)B * feat * 4);
    fc1_acc = take((size_t)B * 1024 * 4);
    fc1d = take((size_t)B * 1024 * 4);
    dfc1 = take((size_t)B * 1024 * 4);
    gA = take(act_numel[0] * 4);
    gB = take(act_numel[0] * 4);
    wrot = take((size_t)9 * 128 * 128 * 4);
    mask1 = take((size_t)B * feat);
    mask2 = take((size_t)B * 1024);
    tc = o;
    o += ((numeric_mode == UDH_NUMERIC_BF16X3 ? x3_workspace_bytes(B, P) : tc_workspace_bytes(B, P, numeric_mode)) + 255) / 256 * 256;
    total = o;
  }
};

template <typename T>
inline T* at(void* ws, size_t off) { return reinterpret_cast<T*>(reinterpret_cast<char*>(ws) + off); }

int check_cnn_args(const char* fn, int B, int P, int numeric_mode) {
  UDH_REQUIRE(B >= 1, "%s: batch must be >= 1", fn);
  UDH_REQUIRE(P >= 128 && P % 128 == 0, "%s: patch size must be a multiple of 128 (got %d)", fn, P);
  UDH_REQUIRE(numeric_mode == UDH_NUMERIC_FP32 || numeric_mode == UDH_NUMERIC_BF16 || numeric_mode == UDH_NUMERIC_BF16X3,
              "%s: unknown numeric_mode %d", fn, numeric_mode);
  UDH_REQUIRE(numeric_mode == UDH_NUMERIC_FP32 || P == 128,
              "%s: the tensor-core modes are tiled for the reference's 128x128 patches (got %d); use UDH_NUMERIC_FP32", fn, P);
  // fc1's weight gradient is an SGEMM with M = (P/8)^2 * 128 rows, one CTA row per 64 of them on grid.y (<= 65535)
  UDH_REQUIRE((size_t)(P / 8) * (P / 8) * 128 / 64 <= 65535,
              "%s: patch size %d is too large: fc1's weight gradient would need %zu CTA rows (max 65535), so P <= 1408", fn, P,
              (size_t)(P / 8) * (P / 8) * 128 / 64);
  return UDH_OK;
}

#define TRY(call)            \
  do {                       \
    int rc__ = (call);       \
    if (rc__ != UDH_OK) return rc__; \
  } while (0)

}  // namespace
}  // namespace udh

using namespace udh;

extern "C" size_t udh_param_total_floats(int P) { return ParamLayout(P).total; }

extern "C" int udh_param_offset(int P, int tensor, size_t* offset_floats, size_t* numel) {
  UDH_REQUIRE(tensor >= 0 && tensor < 20 && offset_floats && numel, "udh_param_offset: bad tensor index %d", tensor);
  ParamLayout L(P);
  *offset_floats = L.off[tensor];
  *numel = L.numel[tensor];
  return UDH_OK;
}

extern "C" size_t udh_cnn_workspace_bytes(int B, int P, int numeric_mode) {
  if (check_cnn_args("udh_cnn_workspace_bytes", B, P, numeric_mode) != UDH_OK) return 0;
  return Workspace(B, P, numeric_mode).total;
}

extern "C" int udh_cnn_workspace_init(void* ws, size_t ws_bytes, int B, int P, int numeric_mode, void* stream) {
  TRY(check_cnn_args("udh_cnn_workspace_init", B, P, numeric_mode));
  Workspace L(B, P, numeric_mode);
  UDH_REQUIRE(ws && ws_bytes >= L.total, "udh_cnn_workspace_init: bad workspace");
  if (numeric_mode == UDH_NUMERIC_BF16) return tc_workspace_init(ws, L.tc, B, P, as_stream(stream));
  if (numeric_mode == UDH_NUMERIC_BF16X3) return x3_workspace_init(ws, L.tc, B, P, as_stream(stream));
  return UDH_OK;
}

extern "C" int udh_cnn_dropout_masks(void* ws, size_t ws_bytes, int B, int P, int numeric_mode, const uint8_t** mask_conv4,
                                     const uint8_t** mask_fc1) {
  TRY(check_cnn_args("udh_cnn_dropout_masks", B, P, numeric_mode));
  Workspace L(B, P, numeric_mode);
  UDH_REQUIRE(ws && ws_bytes >= L.total && mask_conv4 && mask_fc1, "udh_cnn_dropout_masks: bad workspace");
  *mask_conv4 = at<uint8_t>(ws, L.mask1);
  *mask_fc1 = at<uint8_t>(ws, L.mask2);
  return UDH_OK;
}

extern "C" int udh_cnn_activation(void* ws, size_t ws_bytes, int B, int P, int numeric_mode, int layer, const float** ptr,
                                  size_t* numel) {
  TRY(check_cnn_args("udh_cnn_activation", B, P, numeric_mode));
  Workspace L(B, P, numeric_mode);
  UDH_REQUIRE(ws && ws_bytes >= L.total && ptr && numel && layer >= 0 && layer < 12, "udh_cnn_activation: bad arguments");
  *ptr = at<float>(ws, L.act[layer]);
  *numel = L.act_numel[layer];
  return UDH_OK;
}

extern "C" int udh_debug_x3_materialize(void* ws, size_t ws_bytes, int B, int P, size_t* fp32_region_bytes, void* stream) {
  TRY(check_cnn_args("udh_debug_x3_materialize", B, P, UDH_NUMERIC_BF16X3));
  Workspace L(B, P, UDH_NUMERIC_BF16X3);
  UDH_REQUIRE(ws && ws_bytes >= L.total, "udh_debug_x3_materialize: bad workspace");
  if (fp32_region_bytes) *fp32_region_bytes = L.tc;
  return x3_materialize_acts(ws, L.act, L.tc, B, P, as_stream(stream));
}

extern "C" int udh_cnn_fc1_mirror(void* ws, size_t ws_bytes, int B, int P, int numeric_mode, void** mirror, size_t* param_begin,
                                  size_t* count, int* grad_is_stored) {
  TRY(check_cnn_args("udh_cnn_fc1_mirror", B, P, numeric_mode));
  Workspace L(B, P, numeric_mode);
  UDH_REQUIRE(ws && ws_bytes >= L.total && mirror && param_begin && count && grad_is_stored, "udh_cnn_fc1_mirror: bad arguments");
  ParamLayout PL(P);
  *param_begin = PL.off[16];
  *count = (size_t)(P / 8) * (P / 8) * 128 * 1024;
  *mirror = numeric_mode == UDH_NUMERIC_BF16 ? tc_fc1_mirror(ws, L.tc, B, P)
            : numeric_mode == UDH_NUMERIC_BF16X3 ? x3_fc1_mirror(ws, L.tc, B, P) : nullptr;
  *grad_is_stored = numeric_mode != UDH_NUMERIC_FP32 ? 1 : 0;
  return UDH_OK;
}

extern "C" size_t udh_debug_fc1_scratch_bytes(int B, int numeric_mode) {
  if (B < 1) return 0;
  if (numeric_mode == UDH_NUMERIC_BF16) return fc1_region_bytes(B, 128, 1);
  if (numeric_mode == UDH_NUMERIC_BF16X3) return fc1_region_bytes(B, 128, 2);
  return 0;
}

extern "C" int udh_debug_fc1(int numeric_mode, const float* x, const float* w, const float* dy, float* y, float* dW, float* dx,
                             void* scratch, int B, void* stream) {
  UDH_REQUIRE(numeric_mode == UDH_NUMERIC_FP32 || numeric_mode == UDH_NUMERIC_BF16 || numeric_mode == UDH_NUMERIC_BF16X3,
              "udh_debug_fc1: unknown numeric_mode %d", numeric_mode);
  UDH_REQUIRE(B >= 1, "udh_debug_fc1: batch must be >= 1 (got %d)", B);
  UDH_REQUIRE(x && w && y && (dy == nullptr || (dW && dx)) && (numeric_mode == UDH_NUMERIC_FP32 || scratch),
              "udh_debug_fc1: null pointer");
  const int P = 128, feat = (P / 8) * (P / 8) * 128;
  cudaStream_t st = as_stream(stream);
  // the calls of udh_cnn_fwd_ex / udh_cnn_bwd_phase, with the tensor-core region at the start of `scratch`
  UDH_CUDA(cudaMemsetAsync(y, 0, (size_t)B * 1024 * 4, st));
  if (numeric_mode == UDH_NUMERIC_BF16) {
    TRY(tc_fc1_fwd(x, w, y, scratch, 0, B, P, false, st));
    if (dy) TRY(tc_fc1_bwd(dy, dW, dx, scratch, 0, B, P, st));
  } else if (numeric_mode == UDH_NUMERIC_BF16X3) {
    TRY(x3_fc1_fwd(x, w, y, scratch, 0, B, P, false, st));
    if (dy) TRY(x3_fc1_bwd(dy, dW, dx, scratch, 0, B, P, st));
  } else {
    TRY(fc1_fwd_simt(x, w, y, B, feat, st));
    if (dy) TRY(fc1_bwd_simt(x, w, dy, dW, dx, B, feat, st));
  }
  return UDH_OK;
}

extern "C" int udh_debug_fc1_ex(const float* x, const float* w, const float* dy, float* y, float* dW, float* dx, int B, int P,
                                void* stream) {
  TRY(check_cnn_args("udh_debug_fc1_ex", B, P, UDH_NUMERIC_FP32));
  UDH_REQUIRE(x && w && y && (dy == nullptr || (dW && dx)), "udh_debug_fc1_ex: null pointer");
  const int feat = (P / 8) * (P / 8) * 128;
  cudaStream_t st = as_stream(stream);
  // the fp32 calls of udh_cnn_fwd_ex / udh_cnn_bwd_phase at this patch size
  UDH_CUDA(cudaMemsetAsync(y, 0, (size_t)B * 1024 * 4, st));
  TRY(fc1_fwd_simt(x, w, y, B, feat, st));
  if (dy) TRY(fc1_bwd_simt(x, w, dy, dW, dx, B, feat, st));
  return UDH_OK;
}

extern "C" int udh_debug_tc_pool(int numeric_mode, const float* in, float* out, uint32_t* codes, const float* dout, float* din, int B,
                                 int H, int W, int C, void* stream) {
  UDH_REQUIRE(numeric_mode == UDH_NUMERIC_BF16 || numeric_mode == UDH_NUMERIC_BF16X3, "udh_debug_tc_pool: unknown numeric_mode %d",
              numeric_mode);
  UDH_REQUIRE((in || din) && codes && (!in || out) && (!din || dout), "udh_debug_tc_pool: null pointer");
  UDH_REQUIRE(B >= 1 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && C > 0 && C % 8 == 0,
              "udh_debug_tc_pool: needs B >= 1, even H and W and C %% 8 == 0");
  cudaStream_t st = as_stream(stream);
  // the two padded streams of the step (in-shaped and out-shaped), in this mode's format: 2 bytes per limb
  const size_t limbs = numeric_mode == UDH_NUMERIC_BF16X3 ? 2 : 1;
  const size_t in_bytes = (size_t)B * (H + 2) * (W + 2) * C * 2 * limbs, out_bytes = (size_t)B * (H / 2 + 2) * (W / 2 + 2) * C * 2 * limbs;
  void* s = nullptr;
  UDH_CUDA(cudaMallocAsync(&s, in_bytes + out_bytes, st));
  uint16_t* s_in = static_cast<uint16_t*>(s);
  uint16_t* s_out = s_in + in_bytes / 2;
  const cudaError_t e = cudaMemsetAsync(s, 0, in_bytes + out_bytes, st);
  int rc = UDH_ECUDA;
  if (e != cudaSuccess) set_error("udh_debug_tc_pool: cudaMemsetAsync failed: %s", cudaGetErrorString(e));
  else if (numeric_mode == UDH_NUMERIC_BF16X3) rc = x3_debug_pool(in, out, codes, dout, din, s_in, s_out, B, H, W, C, st);
  else rc = tc_debug_pool(in, out, codes, dout, din, s_in, s_out, B, H, W, C, st);
  UDH_CUDA(cudaFreeAsync(s, st));                 // stream-ordered: after the kernels above
  return rc;
}

extern "C" int udh_debug_simt_conv(const float* x, const float* x2, const float* w, const float* bias, const float* mask_src,
                                   float* out, float* wrot, int B, int H, int W, int cin, int cout, int relu, int dgrad,
                                   void* stream) {
  UDH_REQUIRE(x && w && out && (!dgrad || wrot), "udh_debug_simt_conv: null pointer");
  UDH_REQUIRE(!dgrad || (!x2 && !bias && !relu), "udh_debug_simt_conv: the dgrad takes one input, no bias and no ReLU");
  UDH_REQUIRE(B >= 1 && H > 0 && W > 0 && H % 8 == 0 && W % 16 == 0, "udh_debug_simt_conv: needs B >= 1, H % 8 == 0, W % 16 == 0");
  const int kin = dgrad ? cout : cin, kout = dgrad ? cin : cout;
  UDH_REQUIRE(kout > 0 && kout % 64 == 0 && (x2 ? kin == 2 : (kin > 0 && kin % 8 == 0)),
              "udh_debug_simt_conv: unsupported channels (cin %d, cout %d, dgrad %d, two planes %d)", cin, cout, dgrad, x2 != nullptr);
  cudaStream_t st = as_stream(stream);
  // the calls of udh_cnn_fwd (forward) and udh_cnn_bwd_phase (dgrad: rotated weights, no bias, the layer below's ReLU mask)
  if (!dgrad) return conv3x3_simt(x, x2, w, bias, mask_src, out, B, H, W, cin, cout, relu, st);
  TRY(rotate_weights(w, wrot, cin, cout, st));
  return conv3x3_simt(x, nullptr, wrot, nullptr, mask_src, out, B, H, W, cout, cin, 0, st);
}

extern "C" int udh_debug_simt_wgrad(const float* x, const float* x2, const float* g, float* dW, float* db, int B, int H, int W,
                                    int cin, int cout, int* ctas_x, int* tiles_per_cta, int* row_split, void* stream) {
  UDH_REQUIRE(x && g && dW && db, "udh_debug_simt_wgrad: null pointer");
  UDH_REQUIRE(B >= 1 && H > 0 && W > 0 && H % 8 == 0 && W % 16 == 0, "udh_debug_simt_wgrad: needs B >= 1, H % 8 == 0, W % 16 == 0");
  UDH_REQUIRE(cout > 0 && cout % 64 == 0 && (x2 ? cin == 2 : (cin > 0 && cin % 16 == 0)),
              "udh_debug_simt_wgrad: unsupported channels (cin %d, cout %d, two planes %d)", cin, cout, x2 != nullptr);
  const WgradPartition p = wgrad3x3_partition(B, H, W, cin, cout, x2 != nullptr);
  if (ctas_x) *ctas_x = p.ctas_x;
  if (tiles_per_cta) *tiles_per_cta = p.tiles_per_cta;
  if (row_split) *row_split = p.row_split;
  return wgrad3x3_simt(x, x2, g, dW, db, B, H, W, cin, cout, as_stream(stream));
}

extern "C" int udh_debug_simt_pool(const float* in, float* out, const float* dout, float* din, int B, int H, int W, int C,
                                   void* stream) {
  UDH_REQUIRE(in && (out || din) && (!din || dout), "udh_debug_simt_pool: null pointer");
  UDH_REQUIRE(B >= 1 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && C > 0 && C % 4 == 0,
              "udh_debug_simt_pool: needs B >= 1, even H and W and C % 4 == 0");
  cudaStream_t st = as_stream(stream);
  if (out) TRY(maxpool2x2_fwd(in, out, B, H, W, C, st));
  if (din) TRY(maxpool2x2_bwd(in, dout, din, B, H, W, C, st));
  return UDH_OK;
}

extern "C" int udh_cnn_fwd(const float* params, const float* I1, const float* I2, float* h4p, void* ws, size_t ws_bytes,
                           int B, int P, int train, uint64_t seed, int numeric_mode, void* stream) {
  return udh_cnn_fwd_ex(params, I1, I2, h4p, ws, ws_bytes, B, P, train, seed, numeric_mode, 0, stream);
}

extern "C" int udh_cnn_fwd_ex(const float* params, const float* I1, const float* I2, float* h4p, void* ws, size_t ws_bytes,
                              int B, int P, int train, uint64_t seed, int numeric_mode, int flags, void* stream) {
  TRY(check_cnn_args("udh_cnn_fwd", B, P, numeric_mode));
  UDH_REQUIRE(params && I1 && I2 && h4p && ws, "udh_cnn_fwd: null pointer");
  Workspace L(B, P, numeric_mode);
  if (ws_bytes < L.total) { set_error("udh_cnn_fwd: workspace too small (%zu < %zu)", ws_bytes, L.total); return UDH_EWS; }
  ParamLayout PL(P);
  cudaStream_t st = as_stream(stream);
  const int feat = (P / 8) * (P / 8) * 128;

  if (numeric_mode == UDH_NUMERIC_BF16) {
    TRY(tc_cnn_fwd_convs(params, PL.off, I1, I2, ws, L.act, L.tc, B, P, st));
  } else if (numeric_mode == UDH_NUMERIC_BF16X3) {
    TRY(x3_cnn_fwd_convs(params, PL.off, I1, I2, ws, L.act, L.tc, B, P, st));
  } else {
    // conv blocks (homography_model.py:107-118)
    const float* cur0 = I1;
    const float* cur1 = I2;
    for (int i = 0; i < 8; ++i) {
      const int s = P / kConv[i].div;
      {
        ProfScope ps(PROF_CONV_FWD0 + i, st);
        TRY(conv3x3_simt(cur0, cur1, params + PL.off[2 * i], params + PL.off[2 * i + 1], nullptr, at<float>(ws, L.act[i]), B,
                         s, s, kConv[i].cin, kConv[i].cout, 1, st));
      }
      cur0 = at<float>(ws, L.act[i]);
      cur1 = nullptr;
      if (i == 1 || i == 3 || i == 5) {
        const int pi = 8 + i / 2;
        ProfScope ps(PROF_POOL_FWD, st);
        TRY(maxpool2x2_fwd(cur0, at<float>(ws, L.act[pi]), B, s, s, kConv[i].cout, st));
        cur0 = at<float>(ws, L.act[pi]);
      }
    }
  }
  // dropout after conv4_2 (homography_model.py:119-121), flatten NHWC (:124)
  const float* feat_in = at<float>(ws, L.act[7]);
  if (train) {
    ProfScope ps(PROF_ELTWISE, st);
    TRY(dropout_fwd(feat_in, at<float>(ws, L.a4d), at<uint8_t>(ws, L.mask1), (size_t)B * feat, seed, 1, st));
    feat_in = at<float>(ws, L.a4d);
  }
  // fc1 + ReLU + dropout (:126-129): split-K SGEMM into a zeroed accumulator, then the fused epilogue
  ProfScope ps_fc(PROF_FC_FWD, st);
  UDH_CUDA(cudaMemsetAsync(at<float>(ws, L.fc1_acc), 0, (size_t)B * 1024 * 4, st));
  if (numeric_mode == UDH_NUMERIC_BF16) {
    TRY(tc_fc1_fwd(feat_in, params + PL.off[16], at<float>(ws, L.fc1_acc), ws, L.tc, B, P, (flags & UDH_FWD_FC1_MIRROR_CURRENT) != 0, st));
  } else if (numeric_mode == UDH_NUMERIC_BF16X3) {
    TRY(x3_fc1_fwd(feat_in, params + PL.off[16], at<float>(ws, L.fc1_acc), ws, L.tc, B, P, (flags & UDH_FWD_FC1_MIRROR_CURRENT) != 0, st));
  } else {
    TRY(fc1_fwd_simt(feat_in, params + PL.off[16], at<float>(ws, L.fc1_acc), B, feat, st));
  }
  TRY(bias_act_dropout(at<float>(ws, L.fc1_acc), params + PL.off[17], at<float>(ws, L.act[11]), at<float>(ws, L.fc1d),
                       train ? at<uint8_t>(ws, L.mask2) : nullptr, B, 1024, 1, 1, seed, 2, st));
  // fc2, linear (:130-131): K = 1024 split 16 ways (2 CTAs walking K serially were latency bound), atomic accumulation
  UDH_CUDA(cudaMemsetAsync(h4p, 0, (size_t)B * 8 * 4, st));
  TRY(sgemm_simt(at<float>(ws, L.fc1d), 1024, 1, params + PL.off[18], 8, 1, h4p, 8, B, 8, 1024, 16, 0, st));
  TRY(bias_act_dropout(h4p, params + PL.off[19], h4p, nullptr, nullptr, B, 8, 0, 0, 0, 0, st));
  return UDH_OK;
}

extern "C" int udh_cnn_bwd(const float* params, const float* I1, const float* I2, const float* dh4p, float* grads, void* ws,
                           size_t ws_bytes, int B, int P, int train, int numeric_mode, void* stream) {
  return udh_cnn_bwd_phase(params, I1, I2, dh4p, grads, ws, ws_bytes, B, P, train, numeric_mode, UDH_BWD_ALL, stream);
}

extern "C" int udh_cnn_bwd_phase(const float* params, const float* I1, const float* I2, const float* dh4p, float* grads, void* ws,
                                 size_t ws_bytes, int B, int P, int train, int numeric_mode, int phase, void* stream) {
  TRY(check_cnn_args("udh_cnn_bwd", B, P, numeric_mode));
  UDH_REQUIRE(phase == UDH_BWD_ALL || phase == UDH_BWD_HEAD || phase == UDH_BWD_CONVS, "udh_cnn_bwd_phase: bad phase %d", phase);
  UDH_REQUIRE(params && I1 && I2 && dh4p && grads && ws, "udh_cnn_bwd: null pointer");
  Workspace L(B, P, numeric_mode);
  if (ws_bytes < L.total) { set_error("udh_cnn_bwd: workspace too small (%zu < %zu)", ws_bytes, L.total); return UDH_EWS; }
  ParamLayout PL(P);
  cudaStream_t st = as_stream(stream);
  const int feat = (P / 8) * (P / 8) * 128;
  float* gA = at<float>(ws, L.gA);
  float* gB = at<float>(ws, L.gB);
  float* dfc1 = at<float>(ws, L.dfc1);
  float* wrot = at<float>(ws, L.wrot);
  const float* fc1d = at<float>(ws, L.fc1d);
  const float* feat_in = train ? at<float>(ws, L.a4d) : at<float>(ws, L.act[7]);

  if (phase != UDH_BWD_CONVS) {
  // fc2
  prof_begin(PROF_FC_BWD, st);
  TRY(sgemm_simt(fc1d, 1, 1024, dh4p, 8, 1, grads + PL.off[18], 8, 1024, 8, B, 1, 1, st));          // dW2 += fc1d^T . dh4p
  TRY(colsum_accum(dh4p, grads + PL.off[19], B, 8, st));
  TRY(sgemm_simt(dh4p, 8, 1, params + PL.off[18], 1, 8, dfc1, 1024, B, 1024, 8, 1, 0, st));          // dfc1d = dh4p . W2^T
  TRY(drop_relu_bwd(dfc1, train ? at<uint8_t>(ws, L.mask2) : nullptr, at<float>(ws, L.act[11]), (size_t)B * 1024, st));
  // fc1
  if (numeric_mode == UDH_NUMERIC_BF16) {
    TRY(tc_fc1_bwd(dfc1, grads + PL.off[16], gA, ws, L.tc, B, P, st));
  } else if (numeric_mode == UDH_NUMERIC_BF16X3) {
    TRY(x3_fc1_bwd(dfc1, grads + PL.off[16], gA, ws, L.tc, B, P, st));
  } else {
    TRY(fc1_bwd_simt(feat_in, params + PL.off[16], dfc1, grads + PL.off[16], gA, B, feat, st));
  }
  TRY(colsum_accum(dfc1, grads + PL.off[17], B, 1024, st));
  TRY(drop_relu_bwd(gA, train ? at<uint8_t>(ws, L.mask1) : nullptr, at<float>(ws, L.act[7]), (size_t)B * feat, st));
  prof_end(PROF_FC_BWD, st);
  }
  if (phase == UDH_BWD_HEAD) return UDH_OK;

  if (numeric_mode == UDH_NUMERIC_BF16) {
    return tc_cnn_bwd_convs(params, PL.off, I1, I2, grads, gA, gB, ws, L.act, L.tc, B, P, st);
  }
  if (numeric_mode == UDH_NUMERIC_BF16X3) {
    return x3_cnn_bwd_convs(params, PL.off, I1, I2, grads, gA, ws, L.tc, B, P, st);
  }

  // conv stack, top down.  `g` always holds the gradient w.r.t. the PRE-activation output of layer i.
  float* g = gA;
  float* other = gB;
  for (int i = 7; i >= 0; --i) {
    TRY(bwd_marker_record(i, st));
    const int s = P / kConv[i].div;
    const int cin = kConv[i].cin, cout = kConv[i].cout;
    // layer input: previous conv output, a pool output, or the two input planes
    const float* x0;
    const float* x1 = nullptr;
    if (i == 0) { x0 = I1; x1 = I2; }
    else if (i == 2 || i == 4 || i == 6) x0 = at<float>(ws, L.act[8 + (i - 2) / 2]);
    else x0 = at<float>(ws, L.act[i - 1]);
    {
      ProfScope ps(PROF_CONV_WGRAD0 + i, st);
      TRY(wgrad3x3_simt(x0, x1, g, grads + PL.off[2 * i], grads + PL.off[2 * i + 1], B, s, s, cin, cout, st));
    }
    if (i == 0) break;
    const bool below_is_pool = (i == 2 || i == 4 || i == 6);
    {
      ProfScope ps(PROF_CONV_DGRAD0 + i, st);
      TRY(rotate_weights(params + PL.off[2 * i], wrot, cin, cout, st));
      // dgrad: conv over g with the rotated kernel; ReLU mask of the layer below fused unless a pool sits between
      TRY(conv3x3_simt(g, nullptr, wrot, nullptr, below_is_pool ? nullptr : at<float>(ws, L.act[i - 1]), other, B, s, s,
                       cout, cin, 0, st));
    }
    { float* t = g; g = other; other = t; }
    if (below_is_pool) {
      // g = d pool_out  ->  d (pre-activation of conv i-1), arg-max routing + ReLU mask
      ProfScope ps(PROF_POOL_BWD, st);
      TRY(maxpool2x2_bwd(at<float>(ws, L.act[i - 1]), g, other, B, 2 * s, 2 * s, cin, st));
      { float* t = g; g = other; other = t; }
    }
  }
  return UDH_OK;
}
