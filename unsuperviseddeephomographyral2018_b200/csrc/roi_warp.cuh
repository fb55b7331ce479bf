// The ROI warp helpers the mosaic kernels share (warp_perspective.cu) with the graph-cut seams (seam_gc.cu) and the
// seam-scale upscale (seam_scale.cu): cv2's warpPerspective coordinates and taps (the rules: warp_perspective.cu's
// header), a frame on its ROI rectangle and the host helpers that fill and upload its table, and the seam masks' pool
// layout.  The graph-cut seam pass (seam_gc.cu) is declared at the end.
#pragma once
#include <cstdint>
#include <vector>

#include "common.cuh"

namespace udh {

__device__ __forceinline__ void cv_invert3(const double* m, double* t) {
  auto dm = [](double a, double b) { return __dmul_rn(a, b); };
  auto cof = [&](int a, int b, int c, int d) { return __dsub_rn(dm(m[a], m[b]), dm(m[c], m[d])); };
  double det = __dadd_rn(__dsub_rn(dm(m[0], cof(4, 8, 5, 7)), dm(m[1], cof(3, 8, 5, 6))), dm(m[2], cof(3, 7, 4, 6)));
  if (det == 0.0) {
    for (int k = 0; k < 9; ++k) t[k] = 0.0;
    return;
  }
  const double d = __ddiv_rn(1.0, det);
  t[0] = dm(cof(4, 8, 5, 7), d); t[1] = dm(cof(2, 7, 1, 8), d); t[2] = dm(cof(1, 5, 2, 4), d);
  t[3] = dm(cof(5, 6, 3, 8), d); t[4] = dm(cof(0, 8, 2, 6), d); t[5] = dm(cof(2, 3, 0, 5), d);
  t[6] = dm(cof(3, 7, 4, 6), d); t[7] = dm(cof(1, 6, 0, 7), d); t[8] = dm(cof(0, 4, 1, 3), d);
}

__device__ __forceinline__ int wp_fixed(double num, double W) {
  const double f = fmax(-2147483648.0, fmin(2147483647.0, __dmul_rn(num, W)));
  return __double2int_rn(f);
}

// The source position of output pixel (x, y) in 1/32 pixel (X, Y); returns the denominator before 32 / W (0: cv2 lands on
// source pixel (0, 0)).
__device__ __forceinline__ double wp_coords(const double* mi, int x, int y, int bw, int& X, int& Y) {
  const int xb = x - x % bw;
  const double dxb = (double)xb, dy = (double)y, dx1 = (double)(x - xb);
  const double X0 = __dadd_rn(__dadd_rn(__dmul_rn(mi[0], dxb), __dmul_rn(mi[1], dy)), mi[2]);
  const double Y0 = __dadd_rn(__dadd_rn(__dmul_rn(mi[3], dxb), __dmul_rn(mi[4], dy)), mi[5]);
  const double W0 = __dadd_rn(__dadd_rn(__dmul_rn(mi[6], dxb), __dmul_rn(mi[7], dy)), mi[8]);
  const double Wd = __dadd_rn(W0, __dmul_rn(mi[6], dx1));
  const double W = Wd != 0.0 ? __ddiv_rn(32.0, Wd) : 0.0;
  X = wp_fixed(__dadd_rn(X0, __dmul_rn(mi[0], dx1)), W);
  Y = wp_fixed(__dadd_rn(Y0, __dmul_rn(mi[3], dx1)), W);
  return Wd;
}

// The bilinear value at (X, Y) (1/32 pixel) of an h x w source with C channels: 15-bit weights, taps outside read 0.
template <int C>
__device__ __forceinline__ void wp_sample(const uint8_t* __restrict__ s, int h, int w, int X, int Y, int* v) {
  const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767);
  const int fx = X & 31, fy = Y & 31;
  const int wt[4] = {(32 - fx) * (32 - fy) * 32, fx * (32 - fy) * 32, (32 - fx) * fy * 32, fx * fy * 32};
  int acc[C];
#pragma unroll
  for (int c = 0; c < C; ++c) acc[c] = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int tx = sx + (k & 1), ty = sy + (k >> 1);
    if ((unsigned)tx < (unsigned)w && (unsigned)ty < (unsigned)h) {
      const uint8_t* p = s + ((int64_t)ty * w + tx) * C;
#pragma unroll
      for (int c = 0; c < C; ++c) acc[c] += wt[k] * (int)__ldg(p + c);
    }
  }
#pragma unroll
  for (int c = 0; c < C; ++c) v[c] = (acc[c] + (1 << 14)) >> 15;
}

// A frame warped onto its ROI rectangle of the canvas (the multi-band blend's feed, the exposure statistics, the seams):
// the frame, the ROI (rx, ry, rw, rh) and the ROI warp's tile width.  roi_frame fills it on the host.
struct RoiFrame {
  const uint8_t* src;
  int h, w;
  int rx, ry, rw, rh, bw;
};

// Frame (s, h, w)'s ROI warp at ROI pixel (sx, sy) (tile width bw): its value, and whether the pixel is valid.
__device__ __forceinline__ bool mb_roi_warp(const uint8_t* __restrict__ s, int h, int w, const double* mi, int sx, int sy, int bw,
                                            int* v) {
  int X, Y;
  const double Wd = wp_coords(mi, sx, sy, bw, X, Y);
  wp_sample<3>(s, h, w, X, Y, v);
  return Wd != 0.0 && X >= 0 && X <= 32 * (w - 1) && Y >= 0 && Y <= 32 * (h - 1);
}

// ---- host helpers of the ROI-frame entry points ----------------------------------------------------------------------
inline size_t mb_align(size_t v) { return (v + 255) & ~(size_t)255; }

// The warp's tile width for an h x w output: tiles of up to 16 rows and 1024 pixels.
inline int warp_tile_w(int h, int w) {
  const int bh = h < 16 ? h : 16;
  return 1024 / bh < w ? 1024 / bh : w;
}

// Frame k's ROI rois[k] (x_lo, y_lo, x_hi, y_hi: non-empty, inside the dst_h x dst_w canvas) -> F, with the frame's
// pointer and size unless frames and sizes are null (the workspace-size calls leave them unset).  0 or an error.
inline int roi_frame(const uint8_t* const* frames, const int32_t* sizes, const int32_t* rois, int k, int dst_h, int dst_w, RoiFrame& F,
                     const char* what) {
  const int* r = rois + 4 * k;
  UDH_REQUIRE(r[0] >= 0 && r[1] >= 0 && r[0] < r[2] && r[1] < r[3] && r[2] <= dst_w && r[3] <= dst_h,
              "%s: frame %d's ROI (%d, %d)..(%d, %d) is empty or leaves the %dx%d canvas", what, k, r[0], r[1], r[2], r[3], dst_h,
              dst_w);
  F.rx = r[0]; F.ry = r[1]; F.rw = r[2] - r[0]; F.rh = r[3] - r[1];
  F.bw = warp_tile_w(F.rh, F.rw);
  if (frames) {
    UDH_REQUIRE(frames[k], "%s: frame %d is a null pointer", what, k);
    F.src = frames[k];
  }
  if (sizes) {
    F.h = sizes[2 * k];
    F.w = sizes[2 * k + 1];
    UDH_REQUIRE(F.h >= 1 && F.w >= 1 && F.h < 32767 && F.w < 32767, "%s: frame %d is %dx%d", what, k, F.h, F.w);
  }
  return UDH_OK;
}

// Copies a host table to dst on the device (pageable source: the copy is staged before this returns, so the table may go).
template <class T>
inline int upload(void* dst, const std::vector<T>& table, cudaStream_t st, const char* what) {
  const cudaError_t e = cudaMemcpyAsync(dst, table.data(), table.size() * sizeof(T), cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) {
    set_error("%s: table copy: %s", what, cudaGetErrorString(e));
    return UDH_ECUDA;
  }
  return UDH_OK;
}

inline unsigned mb_blocks(int64_t px) {
  const int64_t b = (px + 255) / 256;
  return (unsigned)(b < 1 ? 1 : b > 4096 ? 4096 : b);
}

// ---- seam masks: every fed frame's mask on its ROI (rh x rw bytes at element offset off of a pool) ----------------------
constexpr int SEAM_GAP = 10;      // a pair's window: the ROIs' intersection grown by SEAM_GAP on every side

struct SeamFrame : RoiFrame {
  int64_t off;                  // the ROI's element offset in the mask pools
};

struct SeamRect {                  // a frame's ROI and pool offset, passed by value to the pair kernels
  int64_t off;
  int rx, ry, rw, rh;
};

__device__ __forceinline__ bool seam_at(const uint8_t* __restrict__ seam, const SeamRect& r, int cx, int cy) {
  const int lx = cx - r.rx, ly = cy - r.ry;
  return (unsigned)lx < (unsigned)r.rw && (unsigned)ly < (unsigned)r.rh && seam[r.off + (int64_t)ly * r.rw + lx] != 0;
}

// cv2.detail's GraphCutSeamFinder(COST_COLOR) over the pairs (pi[q], pj[q]) in order (seam_gc.cu): per pair its window
// graph, a maximum flow and the masks' update in the pool seam; the cut values to cut (host, npairs, optional).  fr: the
// frame table on the device (host: its copy), M frame -> ROI; the workspace at base + off, gc_workspace_bytes(off,
// max_win, npairs) in all.  Synchronises.
size_t gc_workspace_bytes(size_t off, int64_t max_win, int64_t npairs);
int gc_seam_pairs(char* base, size_t off, int64_t max_win, const SeamFrame* fr, const std::vector<SeamFrame>& host, const double* M,
                  uint8_t* seam, const std::vector<int>& pi, const std::vector<int>& pj, int64_t* cut, cudaStream_t st, const char* what);

}  // namespace udh
