// Seams at a reduced resolution (cv2's seam_megapix; the rule: oracle/seam_scale.py): the INTER_LINEAR_EXACT resize that
// makes the seam-scale frames (udh_resize_linear_exact_u8), and the upscale of the seam-scale seams to graded blend masks
// on the full-resolution ROIs (udh_mosaic_seam_upscale_u8).  Both sample with 8-bit weights built on the host in float64,
// so no device rounding (FMA contraction included) can move a tap; the sums are integers.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

#include "roi_warp.cuh"

namespace udh {

// ---- INTER_LINEAR_EXACT ------------------------------------------------------------------------------------------------------
// tab (int32): xs0[dw], xs1[dw], xc1[dw], ys0[dh], ys1[dh], yc1[dh] (ops.linear_exact_table): the two taps of each output
// column / row and the upper tap's weight in 1/256 (the lower's is 256 - c1).  One thread per output pixel, all C channels:
// h = c0 p(s0) + c1 p(s1) along both source rows, then (c0' h0 + c1' h1 + 2^15) >> 16 (below 2^24: int32 is exact).
template <int C>
__global__ void __launch_bounds__(256) resize_linear_exact_u8_kernel(const uint8_t* __restrict__ src, const int32_t* __restrict__ tab,
                                                                     uint8_t* __restrict__ dst, int sh, int sw, int dh, int dw) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= dh * dw) return;
  const int dy = o / dw, dx = o - dy * dw;
  const int xs0 = __ldg(tab + dx), xs1 = __ldg(tab + dw + dx), xc1 = __ldg(tab + 2 * dw + dx);
  const int32_t* yt = tab + 3 * dw;
  const int ys0 = __ldg(yt + dy), ys1 = __ldg(yt + dh + dy), yc1 = __ldg(yt + 2 * dh + dy);
  const uint8_t* img = src + (int64_t)blockIdx.y * sh * sw * C;
  const uint8_t* r0 = img + (int64_t)ys0 * sw * C;
  const uint8_t* r1 = img + (int64_t)ys1 * sw * C;
  uint8_t* d = dst + ((int64_t)blockIdx.y * dh * dw + o) * C;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const int h0 = __ldg(r0 + xs0 * C + c) * (256 - xc1) + __ldg(r0 + xs1 * C + c) * xc1;
    const int h1 = __ldg(r1 + xs0 * C + c) * (256 - xc1) + __ldg(r1 + xs1 * C + c) * xc1;
    d[c] = (uint8_t)((h0 * (256 - yc1) + h1 * yc1 + (1 << 15)) >> 16);
  }
}

// ---- the seam masks' upscale ------------------------------------------------------------------------------------------------
// A fed frame: its full-resolution ROI (RoiFrame, the blend pool's offset out), its seam mask on its seam ROI (sx, sy, sw,
// sh on the seam canvas; sw = 0: the seam ROI is empty) and the dilated mask's offset in the workspace pool.
struct UpFrame : RoiFrame {
  int64_t out;
  const uint8_t* seam;
  int sx, sy, sw, sh;
  int64_t dil;
};

// D = cv2.dilate(seam, 3 x 3 rectangle; pixels outside the seam ROI never win) of every frame into the pool.
__global__ void __launch_bounds__(256) seam_dilate_kernel(const UpFrame* __restrict__ fr, uint8_t* __restrict__ pool) {
  const UpFrame* F = fr + blockIdx.y;
  const uint8_t* s = reinterpret_cast<const uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&F->seam)));
  const int sw = __ldg(&F->sw), sh = __ldg(&F->sh), npx = sw * sh;
  uint8_t* D = pool + __ldg(&F->dil);
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < npx; e += gridDim.x * blockDim.x) {
    const int y = e / sw, x = e - y * sw;
    int m = 0;
    for (int dy = max(y - 1, 0); dy <= min(y + 1, sh - 1); ++dy)
      for (int dx = max(x - 1, 0); dx <= min(x + 1, sw - 1); ++dx) m = max(m, (int)__ldg(s + (int64_t)dy * sw + dx));
    D[e] = (uint8_t)m;
  }
}

// Every full-ROI pixel of frame blockIdx.y: its validity (seam_valid_kernel's rule) AND the 4-tap INTER_LINEAR_EXACT sample
// of D at the pixel's canvas position (X, Y) scaled to the seam canvas.  cols [3][dst_w] and rows [3][dst_h] hold the taps
// (s0, s1 on the seam canvas) and the upper weight of every canvas column / row; a tap outside the seam ROI reads 0.
__global__ void __launch_bounds__(256) seam_upscale_kernel(const UpFrame* __restrict__ fr, const double* __restrict__ M,
                                                           const int32_t* __restrict__ cols, const int32_t* __restrict__ rows,
                                                           int dst_w, int dst_h, const uint8_t* __restrict__ pool,
                                                           uint8_t* __restrict__ blend) {
  __shared__ double mi[9];
  const int k = blockIdx.y;
  if (threadIdx.x == 0) cv_invert3(M + (int64_t)k * 9, mi);
  __syncthreads();
  const UpFrame* F = fr + k;
  const int h = __ldg(&F->h), w = __ldg(&F->w), rx = __ldg(&F->rx), ry = __ldg(&F->ry), rw = __ldg(&F->rw), bw = __ldg(&F->bw);
  const int sx = __ldg(&F->sx), sy = __ldg(&F->sy), sw = __ldg(&F->sw), sh = __ldg(&F->sh), npx = rw * __ldg(&F->rh);
  const uint8_t* D = pool + __ldg(&F->dil);
  uint8_t* out = blend + __ldg(&F->out);
  auto at = [&](int ty, int tx) -> int {
    return (unsigned)tx < (unsigned)sw && (unsigned)ty < (unsigned)sh ? (int)__ldg(D + (int64_t)ty * sw + tx) : 0;
  };
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < npx; e += gridDim.x * blockDim.x) {
    const int y = e / rw, x = e - y * rw;
    int X, Y;
    const double Wd = wp_coords(mi, x, y, bw, X, Y);
    int v = 0;
    if (sw > 0 && Wd != 0.0 && X >= 0 && X <= 32 * (w - 1) && Y >= 0 && Y <= 32 * (h - 1)) {
      const int cx = rx + x, cy = ry + y;
      const int t0 = __ldg(cols + cx) - sx, t1 = __ldg(cols + dst_w + cx) - sx, c1 = __ldg(cols + 2 * dst_w + cx);
      const int u0 = __ldg(rows + cy) - sy, u1 = __ldg(rows + dst_h + cy) - sy, d1 = __ldg(rows + 2 * dst_h + cy);
      const int h0 = at(u0, t0) * (256 - c1) + at(u0, t1) * c1;
      const int h1 = at(u1, t0) * (256 - c1) + at(u1, t1) * c1;
      v = (h0 * (256 - d1) + h1 * d1 + (1 << 15)) >> 16;
    }
    out[e] = (uint8_t)v;
  }
}

// The INTER_LINEAR_EXACT taps of canvas axis 0 .. N - 1 on a seam-canvas axis of n pixels, sampled at (X + 1/2) a - 1/2 in
// float64 on the host, into t[0 .. 3N): s0, then s1, then c1 (rint: ties to even, cv2's cvRound).
static void exact_taps(int N, int n, double a, int32_t* t) {
  for (int X = 0; X < N; ++X) {
    const double f = ((double)X + 0.5) * a - 0.5, s = std::floor(f);
    const int si = (int)s, c1 = (int)std::nearbyint((f - s) * 256.0);
    t[X] = si < 0 ? 0 : si + 1 > n - 1 ? n - 1 : si;
    t[N + X] = si < 0 ? 0 : si + 1 > n - 1 ? n - 1 : si + 1;
    t[2 * N + X] = c1;
  }
}

// The host's plan of one upscale call: the frame table and the workspace (frame table, tap tables, dilated pool).
struct UpPlan {
  std::vector<UpFrame> fr;
  int64_t max_px = 0, max_seam = 0;
  size_t off_tab, off_pool, total;
};

static int up_plan(const uint8_t* const* frames, const int32_t* sizes, const int32_t* rois, const uint8_t* const* seams,
                   const int32_t* seam_rois, int n, int seam_h, int seam_w, double scale, int dst_h, int dst_w, UpPlan& p,
                   const char* what) {
  UDH_REQUIRE(rois && seam_rois, "%s: null pointer", what);
  UDH_REQUIRE(n >= 1 && n <= UDH_SEAM_MAX_FRAMES && dst_h >= 1 && dst_w >= 1 && dst_h < 32767 && dst_w < 32767 && seam_h >= 1 &&
                  seam_w >= 1 && seam_h <= dst_h && seam_w <= dst_w,
              "%s: bad dimensions (n %d of at most %d, canvas %dx%d, seam canvas %dx%d)", what, n, UDH_SEAM_MAX_FRAMES, dst_h, dst_w,
              seam_h, seam_w);
  UDH_REQUIRE(scale > 0.0 && scale <= 1.0, "%s: scale must be in (0, 1] (got %g)", what, scale);
  p.fr.assign((size_t)n, UpFrame{});
  int64_t out = 0, dil = 0;
  for (int k = 0; k < n; ++k) {
    UpFrame& F = p.fr[k];
    const int rc = roi_frame(frames, sizes, rois, k, dst_h, dst_w, F, what);
    if (rc != UDH_OK) return rc;
    F.out = out;
    out += (int64_t)F.rw * F.rh;
    p.max_px = std::max(p.max_px, (int64_t)F.rw * F.rh);
    const int* r = seam_rois + 4 * k;
    F.dil = dil;
    if (r[2] <= r[0] || r[3] <= r[1]) continue;                       // no seam ROI: an all-zero mask
    UDH_REQUIRE(r[0] >= 0 && r[1] >= 0 && r[2] <= seam_w && r[3] <= seam_h,
                "%s: frame %d's seam ROI (%d, %d)..(%d, %d) leaves the %dx%d seam canvas", what, k, r[0], r[1], r[2], r[3], seam_h,
                seam_w);
    F.sx = r[0]; F.sy = r[1]; F.sw = r[2] - r[0]; F.sh = r[3] - r[1];
    if (seams) {
      UDH_REQUIRE(seams[k], "%s: frame %d's seam mask is a null pointer", what, k);
      F.seam = seams[k];
    }
    dil += (int64_t)F.sw * F.sh;
    p.max_seam = std::max(p.max_seam, (int64_t)F.sw * F.sh);
  }
  p.off_tab = mb_align((size_t)n * sizeof(UpFrame));
  p.off_pool = mb_align(p.off_tab + 3 * (size_t)(dst_w + dst_h) * sizeof(int32_t));
  p.total = mb_align(p.off_pool + (size_t)dil);
  return UDH_OK;
}

}  // namespace udh

using namespace udh;

extern "C" int udh_resize_linear_exact_u8(const uint8_t* src, const int32_t* tab, uint8_t* dst, int n, int src_h, int src_w, int c,
                                          int dst_h, int dst_w, void* stream) {
  const char* what = "udh_resize_linear_exact_u8";
  UDH_REQUIRE(src && tab && dst, "%s: null pointer", what);
  UDH_REQUIRE(c == 1 || c == 3, "%s: channels must be 1 or 3 (got %d)", what, c);
  UDH_REQUIRE(n >= 0 && n <= 65535 && src_h >= 1 && src_w >= 1 && dst_h >= 1 && dst_w >= 1 && (int64_t)dst_h * dst_w < INT32_MAX &&
                  (int64_t)src_w * c < INT32_MAX,
              "%s: bad dimensions (n %d, %dx%d -> %dx%d)", what, n, src_h, src_w, dst_h, dst_w);
  if (n == 0) return UDH_OK;
  const cudaStream_t st = as_stream(stream);
  const dim3 grid((unsigned)(((int64_t)dst_h * dst_w + 255) / 256), (unsigned)n);
  if (c == 3)
    resize_linear_exact_u8_kernel<3><<<grid, 256, 0, st>>>(src, tab, dst, src_h, src_w, dst_h, dst_w);
  else
    resize_linear_exact_u8_kernel<1><<<grid, 256, 0, st>>>(src, tab, dst, src_h, src_w, dst_h, dst_w);
  return check_launch(what);
}

extern "C" size_t udh_mosaic_seam_upscale_workspace_bytes(const int32_t* rois, const int32_t* seam_rois, int n, int seam_h, int seam_w,
                                                          double scale, int dst_h, int dst_w) {
  UpPlan p;
  return up_plan(nullptr, nullptr, rois, nullptr, seam_rois, n, seam_h, seam_w, scale, dst_h, dst_w, p,
                 "udh_mosaic_seam_upscale_u8") == UDH_OK
             ? p.total
             : 0;
}

extern "C" int udh_mosaic_seam_upscale_u8(const uint8_t* const* frames, const int32_t* sizes, const double* M, const int32_t* rois,
                                          const uint8_t* const* seams, const int32_t* seam_rois, int n, int seam_h, int seam_w,
                                          double scale, int dst_h, int dst_w, uint8_t* blend, void* ws, size_t ws_bytes, void* stream) {
  const char* what = "udh_mosaic_seam_upscale_u8";
  UDH_REQUIRE(frames && sizes && M && seams && blend && ws, "%s: null pointer", what);
  UpPlan p;
  int rc = up_plan(frames, sizes, rois, seams, seam_rois, n, seam_h, seam_w, scale, dst_h, dst_w, p, what);
  if (rc != UDH_OK) return rc;
  if (ws_bytes < p.total) {
    set_error("%s: workspace of %zu bytes, %zu needed", what, ws_bytes, p.total);
    return UDH_EWS;
  }
  std::vector<int32_t> tab(3 * (size_t)(dst_w + dst_h));
  exact_taps(dst_w, seam_w, scale, tab.data());
  exact_taps(dst_h, seam_h, scale, tab.data() + 3 * (size_t)dst_w);
  const cudaStream_t st = as_stream(stream);
  char* base = static_cast<char*>(ws);
  if ((rc = upload(base, p.fr, st, what)) != UDH_OK || (rc = upload(base + p.off_tab, tab, st, what)) != UDH_OK) return rc;
  const UpFrame* fr = reinterpret_cast<const UpFrame*>(base);
  const int32_t* cols = reinterpret_cast<const int32_t*>(base + p.off_tab);
  uint8_t* pool = reinterpret_cast<uint8_t*>(base + p.off_pool);
  if (p.max_seam > 0) {
    seam_dilate_kernel<<<dim3(mb_blocks(p.max_seam), (unsigned)n), 256, 0, st>>>(fr, pool);
    if ((rc = check_launch("udh_mosaic_seam_upscale_u8 (dilate)")) != UDH_OK) return rc;
  }
  seam_upscale_kernel<<<dim3(mb_blocks(p.max_px), (unsigned)n), 256, 0, st>>>(fr, M, cols, cols + 3 * dst_w, dst_w, dst_h, pool, blend);
  return check_launch(what);
}
