// The report image of the reference's test harnesses (code/utils/utils.py:209-307, save_correspondences_img), batched:
//   draw_lut_kernel    denorm_u8 tabulated per (sample, image, channel)
//   draw_fill_kernel   one thread per canvas pixel: [left image | right image]
//   draw_prims_kernel  one CTA per sample draws the primitives in the reference's order, with a barrier wherever the
//                      next primitive may read or overwrite what the previous one wrote:
//                        the prediction polygon (thick 3, LINE_8) clipped to the right image, the two thick GT polygons,
//                        then per match: a LINE_AA line and two LINE_AA circles of radius 7 (12 segments each).
// The integer arithmetic is cv2's (drawing.cpp of OpenCV 4.x, pinned black-box by tests/test_draw_oracle.py against
// oracle/draw.py): int32 points, int64 16.16 fixed point, the double-precision intercepts of clipLine, the int32 wraps of
// cv2's casts.  Inside one primitive the work is split over the CTA's threads: constant-colour pixels are set in any
// order, and one LineAA segment blends each pixel at most once (every step has its own major coordinate).
#include <climits>

#include "common.cuh"

namespace udh {

namespace {

constexpr int kDrawThreads = 256;
constexpr int kShift = 16;
constexpr long long kOne = 1ll << kShift;

__constant__ uint8_t kSlopeCorr[32] = {181, 181, 181, 182, 182, 183, 184, 185, 187, 188, 190, 192, 194, 196, 198, 201,
                                       203, 206, 209, 211, 214, 218, 221, 224, 227, 231, 235, 238, 242, 246, 250, 254};
__constant__ uint8_t kFilter[64] = {168, 177, 185, 194, 202, 210, 218, 224, 231, 236, 241, 246, 249, 252, 254, 254,
                                    254, 254, 252, 249, 246, 241, 236, 231, 224, 218, 210, 202, 194, 185, 177, 168,
                                    158, 149, 140, 131, 122, 114, 105, 97, 89, 82, 75, 68, 62, 56, 50, 45,
                                    40, 36, 32, 28, 25, 22, 19, 16, 14, 12, 11, 9, 8, 7, 5, 5};
// utils/utils.py:213-217, 263-264: the colours as cv2 receives them (channel 0, 1, 2)
__constant__ uint8_t kColors[6][3] = {{5, 225, 225}, {2, 10, 240}, {255, 102, 255}, {51, 153, 255}, {102, 255, 255}, {255, 255, 0}};

__device__ __forceinline__ int i32(long long v) { return (int)(unsigned)(unsigned long long)v; }
__device__ __forceinline__ long long wadd(long long a, long long b) {
  return (long long)((unsigned long long)a + (unsigned long long)b);
}
__device__ __forceinline__ long long wmul(long long a, long long b) {
  return (long long)((unsigned long long)a * (unsigned long long)b);
}
// cvRound(double) on x86-64 (cvtsd2si): half to even, NaN / out of int32 -> INT_MIN
__device__ __forceinline__ int cv_round(double d) {
  if (!(d >= -2147483648.5 && d < 2147483647.5)) return INT_MIN;
  return __double2int_rn(d);
}
// (int64)((double)a * (double)b / (double)c), one rounding per operation as on the host
__device__ __forceinline__ long long muldiv(long long a, long long b, long long c) {
  return (long long)__ddiv_rn(__dmul_rn((double)a, (double)b), (double)c);
}

// A drawable rectangle of the canvas: pixel (x, y) is at base + y*pitch + (x0 + x)*3.
struct View {
  uint8_t* base;
  int pitch, x0, w, h;
  __device__ uint8_t* px(int x, int y) const { return base + (size_t)y * pitch + (size_t)(x0 + x) * 3; }
  __device__ void put(int x, int y, const uint8_t* c) const {
    if (x >= 0 && x < w && y >= 0 && y < h) {
      uint8_t* p = px(x, y);
      p[0] = c[0]; p[1] = c[1]; p[2] = c[2];
    }
  }
  __device__ void hline(int y, int xl, int xr, const uint8_t* c) const {   // xl, xr already inside [0, w)
    for (int x = xl; x <= xr; ++x) { uint8_t* p = px(x, y); p[0] = c[0]; p[1] = c[1]; p[2] = c[2]; }
  }
};

// clipLine(Size2l, Point2l&, Point2l&)
__device__ bool clip_line(long long w, long long h, long long& x1, long long& y1, long long& x2, long long& y2) {
  if (w <= 0 || h <= 0) return false;
  const long long right = w - 1, bottom = h - 1;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    long long a;
    if (c1 & 12) {
      a = c1 < 8 ? 0 : bottom;
      x1 += muldiv(a - y1, x2 - x1, y2 - y1);
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      a = c2 < 8 ? 0 : bottom;
      x2 += muldiv(a - y2, x2 - x1, y2 - y1);
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        a = c1 == 1 ? 0 : right;
        y1 += muldiv(a - x1, y2 - y1, x2 - x1);
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        a = c2 == 1 ? 0 : right;
        y2 += muldiv(a - x2, y2 - y1, x2 - x1);
        x2 = a;
        c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

// Line2: the 16.16 LINE_8 rasteriser of FillConvexPoly's outline; pixel k = -1 is the rounded end point
__device__ void line2(const View& v, long long x1, long long y1, long long x2, long long y2, const uint8_t* c, int tid, int nt) {
  if (!clip_line((long long)v.w << kShift, (long long)v.h << kShift, x1, y1, x2, y2)) return;
  long long dx = x2 - x1, dy = y2 - y1;
  const long long ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy;
  const bool horiz = ax > ay;
  long long step;
  int ecount;
  if (horiz) {
    if (dx < 0) { long long t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; dy = -dy; }
    step = (dy << kShift) / (ax | 1);
    ecount = (int)((x2 - x1) >> kShift);
  } else {
    if (dy < 0) { long long t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; dx = -dx; }
    step = (dx << kShift) / (ay | 1);
    ecount = (int)((y2 - y1) >> kShift);
  }
  x1 += kOne >> 1;
  y1 += kOne >> 1;
  for (int k = tid - 1; k <= ecount; k += nt) {
    if (k < 0) {
      v.put(i32((x2 + (kOne >> 1)) >> kShift), i32((y2 + (kOne >> 1)) >> kShift), c);
    } else if (horiz) {
      v.put(i32((x1 >> kShift) + k), i32((y1 + k * step) >> kShift), c);
    } else {
      v.put(i32((x1 + k * step) >> kShift), i32((y1 >> kShift) + k), c);
    }
  }
}

// FillConvexPoly(4 vertices in 16.16, LINE_8, shift 16).  Every thread replays the edge events (at most one per vertex)
// and fills the rows r with r % nt == tid; between events the edges step in closed form x + k*dx, wrapping as cv2's
// repeated int64 additions do.
__device__ void fill_convex4(const View& v, const long long (*p)[2], const uint8_t* c, int tid, int nt) {
  const int n = 4;
  const long long delta = kOne >> 1;
  long long xmin = p[0][0], xmax = p[0][0], ymin = p[0][1], ymax = p[0][1];
  int imin = 0;
  for (int i = 0; i < n; ++i) {
    const long long x = p[i][0], y = p[i][1];
    if (y < ymin) { ymin = y; imin = i; }
    ymax = max(ymax, y); xmax = max(xmax, x); xmin = min(xmin, x);
    const int j = (i + n - 1) % n;
    line2(v, p[j][0], p[j][1], x, y, c, tid, nt);
  }
  xmin = (xmin + delta) >> kShift; xmax = (xmax + delta) >> kShift;
  ymin = (ymin + delta) >> kShift; ymax = (ymax + delta) >> kShift;
  if (i32(xmax) < 0 || i32(ymax) < 0 || i32(xmin) >= v.w || i32(ymin) >= v.h) return;
  ymax = min(ymax, (long long)v.h - 1);
  const int ylast = i32(ymax);
  int edges = n;
  int e_idx[2] = {imin, imin}, e_di[2] = {1, n - 1}, e_ye[2];
  long long e_x[2] = {-kOne, -kOne}, e_dx[2] = {0, 0};
  int y = i32(ymin);
  e_ye[0] = e_ye[1] = y;
  for (;;) {
    for (int i = 0; i < 2; ++i) {
      if (y >= e_ye[i]) {
        int idx0 = e_idx[i], di = e_di[i];
        int idx = idx0 + di;
        if (idx >= n) idx -= n;
        for (; edges-- > 0;) {
          const int ty = i32((p[idx][1] + delta) >> kShift);
          if (ty > y) {
            const long long xs = p[idx0][0], xe = p[idx][0];
            e_ye[i] = ty;
            e_dx[i] = ((xe - xs) * 2 + ((long long)ty - y)) / (2 * ((long long)ty - y));
            e_x[i] = xs;
            e_idx[i] = idx;
            break;
          }
          idx0 = idx;
          idx += di;
          if (idx >= n) idx -= n;
        }
      }
    }
    if (edges < 0) return;
    const long long stop = min(min((long long)e_ye[0], (long long)e_ye[1]), (long long)ylast + 1);
    long long r0 = y < 0 ? 0 : y;
    r0 += ((tid - r0) % nt + nt) % nt;
    for (long long r = r0; r < stop; r += nt) {
      const long long k = r - y;
      long long xa = wadd(e_x[0], wmul(k, e_dx[0])), xb = wadd(e_x[1], wmul(k, e_dx[1]));
      if (xa > xb) { const long long t = xa; xa = xb; xb = t; }
      int xx1 = i32(wadd(xa, delta) >> kShift), xx2 = i32(wadd(xb, delta) >> kShift);
      if (xx2 >= 0 && xx1 < v.w) v.hline((int)r, max(xx1, 0), min(xx2, v.w - 1), c);
    }
    e_x[0] = wadd(e_x[0], wmul(stop - y, e_dx[0]));
    e_x[1] = wadd(e_x[1], wmul(stop - y, e_dx[1]));
    if (stop > ylast) return;
    y = (int)stop;
  }
}

// Circle(fill = 1) of radius r: Bresenham spans with int32 wrap of the span ends
__device__ void circle_fill(const View& v, int cx, int cy, int r, const uint8_t* c) {
  int err = 0, dx = r, dy = 0, plus = 1, minus = (r << 1) - 1;
  while (dx >= dy) {
    const int y11 = i32((long long)cy - dy), y12 = i32((long long)cy + dy), y21 = i32((long long)cy - dx), y22 = i32((long long)cy + dx);
    int x11 = i32((long long)cx - dx), x12 = i32((long long)cx + dx), x21 = i32((long long)cx - dy), x22 = i32((long long)cx + dy);
    if (x11 < v.w && x12 >= 0 && y21 < v.h && y22 >= 0) {
      x11 = max(x11, 0); x12 = min(x12, v.w - 1);
      if ((unsigned)y11 < (unsigned)v.h) v.hline(y11, x11, x12, c);
      if ((unsigned)y12 < (unsigned)v.h) v.hline(y12, x11, x12, c);
      if (x21 < v.w && x22 >= 0) {
        x21 = max(x21, 0); x22 = min(x22, v.w - 1);
        if ((unsigned)y21 < (unsigned)v.h) v.hline(y21, x21, x22, c);
        if ((unsigned)y22 < (unsigned)v.h) v.hline(y22, x21, x22, c);
      }
    }
    dy++;
    err += plus;
    plus += 2;
    const int mask = (err <= 0) - 1;
    err -= minus & mask;
    dx += mask;
    minus -= mask & 2;
  }
}

// ThickLine(thickness 3, LINE_8, shift 0): clip to the view grown by the thickness, widen into a 4-vertex polygon, and
// (cap) a filled radius-2 circle at the second point.  No barrier inside: all of it is one colour.
__device__ void thick3(const View& v, int px0, int py0, int px1, int py1, bool cap, const uint8_t* c, int tid, int nt) {
  const int m = 3;
  long long ax = (long long)px0 + m, ay = (long long)py0 + m, bx = (long long)px1 + m, by = (long long)py1 + m;
  if (!clip_line(v.w + 2 * m, v.h + 2 * m, ax, ay, bx, by)) return;
  const long long x0 = (ax - m) * kOne, y0 = (ay - m) * kOne, x1 = (bx - m) * kOne, y1 = (by - m) * kOne;
  const double dxf = __dmul_rn((double)(x0 - x1), 1.0 / kOne), dyf = __dmul_rn((double)(y1 - y0), 1.0 / kOne);
  double r = __dadd_rn(__dmul_rn(dxf, dxf), __dmul_rn(dyf, dyf));
  const long long th = (long long)m << (kShift - 1);
  if (fabs(r) > 2.220446049250313e-16) {
    r = __ddiv_rn(__dadd_rn((double)th, (double)(kOne / 2)), __dsqrt_rn(r));
    const long long dpx = cv_round(__dmul_rn(dyf, r)), dpy = cv_round(__dmul_rn(dxf, r));
    const long long poly[4][2] = {{x0 + dpx, y0 + dpy}, {x0 - dpx, y0 - dpy}, {x1 - dpx, y1 - dpy}, {x1 + dpx, y1 + dpy}};
    fill_convex4(v, poly, c, tid, nt);
  }
  if (cap && tid == 0) circle_fill(v, i32((x1 + (kOne >> 1)) >> kShift), i32((y1 + (kOne >> 1)) >> kShift), (int)((th + (kOne >> 1)) >> kShift), c);
}

// cv2.polylines(closed, thickness 3): edges v[3]->v[0], v[0]->v[1], ..., each capped at its second vertex
__device__ void polyline3(const View& v, const int* pts, const uint8_t* c, int tid, int nt) {
  for (int e = 0; e < 4; ++e) {
    const int j = (e + 3) & 3;
    thick3(v, pts[2 * j], pts[2 * j + 1], pts[2 * e], pts[2 * e + 1], true, c, tid, nt);
  }
}

__device__ __forceinline__ int blend(int v, int c, int a) {
  v += ((c - v) * a + 127) >> 8;
  v += ((c - v) * a + 127) >> 8;
  return v;
}

// LineAA on 16.16 points: each thread takes the steps s with s % nt == tid; a barrier after the segment.
__device__ void line_aa(const View& v, long long x1, long long y1, long long x2, long long y2, const uint8_t* c, int tid, int nt) {
  if (clip_line((long long)v.w << kShift, (long long)v.h << kShift, x1, y1, x2, y2)) {
    long long dx = x2 - x1, dy = y2 - y1;
    const long long ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy;
    const bool horiz = ax > ay;
    long long step, major, minor;
    int ecount, fi, fj;
    if (horiz) {
      if (dx < 0) { long long t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; dy = -dy; }
      step = (dy << kShift) / (ax | 1);
      x2 += kOne;
      ecount = (int)((x2 >> kShift) - (x1 >> kShift));
      const long long j = -(x1 & (kOne - 1));
      y1 += ((step * j) >> kShift) + (kOne >> 1);
      fi = (int)((x1 >> (kShift - 7)) & 0x78); fj = (int)((x2 >> (kShift - 7)) & 0x78);
      major = x1 >> kShift; minor = y1;
    } else {
      if (dy < 0) { long long t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; dx = -dx; }
      step = (dx << kShift) / (ay | 1);
      y2 += kOne;
      ecount = (int)((y2 >> kShift) - (y1 >> kShift));
      const long long j = -(y1 & (kOne - 1));
      x1 += ((step * j) >> kShift) + (kOne >> 1);
      fi = (int)((y1 >> (kShift - 7)) & 0x78); fj = (int)((y2 >> (kShift - 7)) & 0x78);
      major = y1 >> kShift; minor = x1;
    }
    int slope = (int)((step >> (kShift - 5)) & 0x3f);
    slope ^= step < 0 ? 0x3f : 0;
    slope = (slope & 0x20) ? 0x100 : kSlopeCorr[slope];
    const int t0 = slope << 7, t1 = ((0x78 - fi) | 4) * slope, t2 = (fj | 4) * slope;
    int ep[9];
    ep[0] = 0;
    ep[8] = slope;
    ep[1] = ep[3] = ((((fj - fi) & 0x78) | 4) * slope >> 8) & 0x1ff;
    ep[2] = (t1 >> 8) & 0x1ff;
    ep[4] = ((((fj - fi) + 0x80) | 4) * slope >> 8) & 0x1ff;
    ep[5] = ((t1 + t0) >> 8) & 0x1ff;
    ep[6] = (t2 >> 8) & 0x1ff;
    ep[7] = ((t2 + t0) >> 8) & 0x1ff;
    const int smaj = horiz ? v.w : v.h, smin = horiz ? v.h : v.w;
    for (int s = tid; s <= ecount; s += nt) {
      const int ec = ecount - s;
      const int mj = i32(major + s);
      if ((unsigned)mj >= (unsigned)smaj) continue;
      const long long pos = minor + (long long)s * step;
      const int q = i32((pos >> kShift) - 1);
      const int corr = ep[(((s >= 2) + 1) & (s | 2)) * 3 + (((ec >= 2) + 1) & (ec | 2))];
      const int dist = (int)((pos >> (kShift - 5)) & 31);
      const int f[3] = {kFilter[dist + 32], kFilter[dist], kFilter[63 - dist]};
#pragma unroll
      for (int o = 0; o < 3; ++o) {
        if ((unsigned)(q + o) < (unsigned)smin) {
          const int a = (corr * f[o] >> 8) & 0xff;
          uint8_t* p = horiz ? v.px(mj, q + o) : v.px(q + o, mj);
          p[0] = (uint8_t)blend(p[0], c[0], a);
          p[1] = (uint8_t)blend(p[1], c[1], a);
          p[2] = (uint8_t)blend(p[2], c[2], a);
        }
      }
    }
  }
  __syncthreads();
}

// cv2.circle(centre, 7, thickness 1, LINE_AA): ellipse2Poly with delta 30 (13 vertices, the first repeated last, from
// SinTable), each vertex rounded to 16.16 in cv2's two parts, repeats dropped; one LineAA per consecutive pair.
__device__ void circle_aa7(const View& v, int cx, int cy, const uint8_t* c, int tid, int nt) {
  const float sin30[13] = {0.0f, 0.5f, 0.8660254f, 1.0f, 0.8660254f, 0.5f, 0.0f, -0.5f, -0.8660254f, -1.0f, -0.8660254f, -0.5f, 0.0f};
  const double cxd = (double)((long long)cx * kOne), cyd = (double)((long long)cy * kOne), ad = (double)(7 * kOne);
  long long px = 0, py = 0;
  bool have = false;
  for (int k = 0; k < 13; ++k) {
    const double x = __dmul_rn(ad, (double)sin30[(k + 3) % 12]);     // SinTable[450 - 30k] = cos 30k
    const double y = __dmul_rn(ad, (double)sin30[k]);                                                 // SinTable[30k]
    const double fx = __dsub_rn(__dadd_rn(cxd, __dmul_rn(x, 1.0)), __dmul_rn(y, 0.0));
    const double fy = __dadd_rn(__dadd_rn(cyd, __dmul_rn(x, 0.0)), __dmul_rn(y, 1.0));
    long long qx = (long long)cv_round(__dmul_rn(fx, 1.0 / kOne)) * kOne;
    long long qy = (long long)cv_round(__dmul_rn(fy, 1.0 / kOne)) * kOne;
    qx += cv_round(__dsub_rn(fx, (double)qx));
    qy += cv_round(__dsub_rn(fy, (double)qy));
    if (have && (qx != px || qy != py)) line_aa(v, px, py, qx, qy, c, tid, nt);
    if (!have || qx != px || qy != py) { px = qx; py = qy; }
    have = true;
  }
}

__global__ void __launch_bounds__(256) draw_lut_kernel(const float* __restrict__ aug, uint8_t* __restrict__ lut) {
  const int b = blockIdx.x;
  const bool on = aug && aug[b * 11] != 0.0f;
  for (int i = threadIdx.x; i < 2 * 3 * 256; i += blockDim.x) {
    const int im = i / 768, c = (i / 256) % 3, x = i & 255;
    lut[(size_t)b * 1536 + i] = denorm_u8(x, c, on ? aug + b * 11 + 1 + im * 5 : nullptr);
  }
}

// out[b, y, x] = x < w ? left[b, y, x] : right[b, y, x - w], through the sample's tables
__global__ void __launch_bounds__(256) draw_fill_kernel(const uint8_t* __restrict__ I, const uint8_t* __restrict__ Ip,
                                                        const uint8_t* __restrict__ lut, int prime_left, uint8_t* __restrict__ out,
                                                        int h, int w) {
  const int b = blockIdx.y;
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= h * 2 * w) return;
  const int y = o / (2 * w), x = o - y * 2 * w;
  const bool left = x < w;
  const int im = left == (prime_left != 0) ? 1 : 0;                      // 0: I, 1: I'
  const uint8_t* src = (im ? Ip : I) + (((size_t)b * h + y) * w + (left ? x : x - w)) * 3;
  const uint8_t* t = lut + (size_t)b * 1536 + im * 768;
  uint8_t* d = out + ((size_t)b * h * 2 * w + o) * 3;
  d[0] = t[src[0]];
  d[1] = t[256 + src[1]];
  d[2] = t[512 + src[2]];
}

// verts [B,20,2]: prediction polygon (right-image coordinates), kp2, kp1, line starts, line ends (canvas coordinates)
__global__ void __launch_bounds__(kDrawThreads) draw_prims_kernel(const int* __restrict__ verts, uint8_t* __restrict__ out, int h, int w) {
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  __shared__ int pv[40];
  if (tid < 40) pv[tid] = verts[b * 40 + tid];
  __syncthreads();
  uint8_t* base = out + (size_t)b * h * 2 * w * 3;
  const View right{base, 2 * w * 3, w, w, h}, canvas{base, 2 * w * 3, 0, 2 * w, h};
  polyline3(right, pv, kColors[0], tid, nt);               // on img2 alone, before stacking: clipped to it
  __syncthreads();
  polyline3(canvas, pv + 8, kColors[1], tid, nt);
  polyline3(canvas, pv + 16, kColors[1], tid, nt);
  __syncthreads();
  for (int i = 0; i < 4; ++i) {
    const int* e1 = pv + 24 + 2 * i;
    const int* e2 = pv + 32 + 2 * i;
    line_aa(canvas, (long long)e1[0] * kOne, (long long)e1[1] * kOne, (long long)e2[0] * kOne, (long long)e2[1] * kOne, kColors[2 + i], tid, nt);
    circle_aa7(canvas, e1[0], e1[1], kColors[2 + i], tid, nt);
    circle_aa7(canvas, e2[0], e2[1], kColors[2 + i], tid, nt);
  }
}

}  // namespace

}  // namespace udh

using namespace udh;

extern "C" size_t udh_draw_report_workspace_bytes(int B) { return B >= 1 ? (size_t)B * 1536 : 0; }

extern "C" int udh_draw_report_u8(const uint8_t* I, const uint8_t* I_prime, const float* aug, int prime_left, const int32_t* verts,
                                  uint8_t* out, void* ws, size_t ws_bytes, int B, int img_h, int img_w, void* stream) {
  UDH_REQUIRE(I && I_prime && verts && out && ws, "udh_draw_report_u8: null pointer");
  UDH_REQUIRE(B >= 1 && B <= 65535 && img_h >= 1 && img_w >= 1 && (long long)img_h * img_w <= (1 << 28),
              "udh_draw_report_u8: bad dimensions (B %d, %dx%d)", B, img_h, img_w);
  UDH_REQUIRE(ws_bytes >= udh_draw_report_workspace_bytes(B), "udh_draw_report_u8: workspace of %zu bytes, %zu needed", ws_bytes,
              udh_draw_report_workspace_bytes(B));
  cudaStream_t st = as_stream(stream);
  ProfScope ps(PROF_ELTWISE, st);
  uint8_t* lut = static_cast<uint8_t*>(ws);
  draw_lut_kernel<<<B, 256, 0, st>>>(aug, lut);
  int rc = check_launch("udh_draw_report_u8 (tables)");
  if (rc != UDH_OK) return rc;
  const int npx = img_h * 2 * img_w;
  draw_fill_kernel<<<dim3((npx + 255) / 256, B), 256, 0, st>>>(I, I_prime, lut, prime_left, out, img_h, img_w);
  rc = check_launch("udh_draw_report_u8 (canvas)");
  if (rc != UDH_OK) return rc;
  draw_prims_kernel<<<B, kDrawThreads, 0, st>>>(verts, out, img_h, img_w);
  return check_launch("udh_draw_report_u8 (primitives)");
}
