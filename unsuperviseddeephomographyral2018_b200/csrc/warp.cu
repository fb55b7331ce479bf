// Fused homography spatial-transformer warp + photometric reductions (Rows W and L).
// Reference: code/homography_model.py:252-269 (H' = M^-1 H M, transformer, channel mean, patch gather),
// code/utils/tf_spatial_transformer.py:76-247 (linspace grid, t_s epsilon rule, clip-then-weight bilinear),
// code/homography_model.py:291-296,328 (rec / l1 / l1_smooth / ncc reductions).
//
// The reference materialises a [B,3,H*W] grid, four [B*H*W,C] gathers and a [B,H,W,C] warped image, then keeps
// P*P gray values per sample.  Here coordinates are analytic, only the gathered window is evaluated, the channel
// mean and all loss reductions happen in registers, and HBM sees: one read of the source texels the window
// touches, one read of I2, (optionally) one write of pred_I2.  The kernel is HBM/latency bound — no tensor cores.
#include "common.cuh"

namespace udh {

struct Homog {
  float h[9];       // normalised H' = M^-1 H M (row-major)
  float step_x, step_y;
};

// H' = (M^-1 . H) . M in fp32, in the reference's association order (homography_model.py:254).
// M = [[W/2,0,W/2],[0,Hh/2,Hh/2],[0,0,1]] (fp32, :63-67); M^-1 = [[2/W,0,-1],[0,2/Hh,-1],[0,0,1]] rounded to fp32 (:69-70).
__device__ __forceinline__ void normalise_h(const float* __restrict__ Hp, int img_w, int img_h, Homog& o) {
  const float sx = 0.5f * (float)img_w, sy = 0.5f * (float)img_h;
  const float ix = 1.0f / sx, iy = 1.0f / sy;
  float t[9];
  // T = Minv . H
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    t[c] = fmaf(ix, Hp[c], -Hp[6 + c]);
    t[3 + c] = fmaf(iy, Hp[3 + c], -Hp[6 + c]);
    t[6 + c] = Hp[6 + c];
  }
  // H' = T . M : column 0 scaled by sx, column 1 by sy, column 2 = sx*t0 + sy*t1 + t2
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    o.h[3 * r + 0] = t[3 * r + 0] * sx;
    o.h[3 * r + 1] = t[3 * r + 1] * sy;
    o.h[3 * r + 2] = fmaf(t[3 * r + 0], sx, fmaf(t[3 * r + 1], sy, t[3 * r + 2]));
  }
}

struct Tap {
  int i00, i01, i10, i11;   // flat pixel offsets (y0,x0) (y0,x1) (y1,x0) (y1,x1) within one image
  float wa, wb, wc, wd;     // weights of (y0,x0) (y1,x0) (y0,x1) (y1,x1) — reference naming
  float x, y, x0f, x1f, y0f, y1f;
  float xn, yn, ts;
};

// Clip-then-weight bilinear taps of the source position (x, y) in pixels (tf_spatial_transformer.py:97-137).
__device__ __forceinline__ void tap_from_xy(float x, float y, int W, int Hh, Tap& t) {
  // floor -> int32 with saturation (far-away samples all clip to the border pixel pair anyway)
  const float xf = fminf(fmaxf(floorf(x), -2.0f), (float)W + 1.0f);
  const float yf = fminf(fmaxf(floorf(y), -2.0f), (float)Hh + 1.0f);
  int x0 = (int)xf, y0 = (int)yf;
  if (!(x == x)) x0 = 0;                                     // NaN coordinates: keep indices in range
  if (!(y == y)) y0 = 0;
  int x1 = x0 + 1, y1 = y0 + 1;
  x0 = min(max(x0, 0), W - 1); x1 = min(max(x1, 0), W - 1);
  y0 = min(max(y0, 0), Hh - 1); y1 = min(max(y1, 0), Hh - 1);
  t.x0f = (float)x0; t.x1f = (float)x1; t.y0f = (float)y0; t.y1f = (float)y1;
  t.wa = __fmul_rn(t.x1f - x, t.y1f - y);
  t.wb = __fmul_rn(t.x1f - x, y - t.y0f);
  t.wc = __fmul_rn(x - t.x0f, t.y1f - y);
  t.wd = __fmul_rn(x - t.x0f, y - t.y0f);
  t.i00 = y0 * W + x0; t.i01 = y0 * W + x1; t.i10 = y1 * W + x0; t.i11 = y1 * W + x1;
  t.x = x; t.y = y;
}

// Source coordinates of output grid point (xt, yt) in [-1,1] units, reference semantics
// (tf_spatial_transformer.py:213-240 then _interpolate :97-137).
__device__ __forceinline__ void sample_setup(const Homog& hm, float xt, float yt, int W, int Hh, Tap& t) {
  const float xs = fmaf(hm.h[0], xt, fmaf(hm.h[1], yt, hm.h[2]));
  const float ys = fmaf(hm.h[3], xt, fmaf(hm.h[4], yt, hm.h[5]));
  float ts = fmaf(hm.h[6], xt, fmaf(hm.h[7], yt, hm.h[8]));
  if (!(fabsf(ts) >= 1e-7f)) ts += 1e-6f;                    // smallers = 1e-6 * (1 - [|t| >= 1e-7])
  const float xn = xs / ts, yn = ys / ts;
  const float x = (xn + 1.0f) * (float)W / 2.0f;
  const float y = (yn + 1.0f) * (float)Hh / 2.0f;
  tap_from_xy(x, y, W, Hh, t);
  t.x = x; t.y = y; t.xn = xn; t.yn = yn; t.ts = ts;
}

// ((wa*Ia + wb*Ib) + wc*Ic) + wd*Id with every product and sum rounded separately — the reference evaluates
// four tf.multiply and one add_n (tf_spatial_transformer.py:134-138).  The "black border" cancels exactly only when y
// clips (alone or with x): then Ia == Ib, Ic == Id, wb == -wa and wd == -wc, so wa*Ia + wb*Ib == 0 and the sum is
// exactly 0.  Where only x clips, wa*Ia == -(wc*Ic) and wb*Ib == -(wd*Id), but fl(wa*Ia + wb*Ib) - wa*Ia need not
// equal wb*Ib, so a residue of the blend's rounding, ulp(w*I), can remain (tests/test_gpu_photometric.py bounds it).  A fused multiply-add would leave
// such residues everywhere.
__device__ __forceinline__ float bilinear_rn(const Tap& t, float Ia, float Ib, float Ic, float Id) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(t.wa, Ia), __fmul_rn(t.wb, Ib)), __fmul_rn(t.wc, Ic)), __fmul_rn(t.wd, Id));
}

template <int C>
__device__ __forceinline__ float sample_gray(const float* __restrict__ img, const Tap& t) {
  float acc = 0.f;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const float Ia = __ldg(img + (size_t)t.i00 * C + c), Ib = __ldg(img + (size_t)t.i10 * C + c);
    const float Ic = __ldg(img + (size_t)t.i01 * C + c), Id = __ldg(img + (size_t)t.i11 * C + c);
    acc = __fadd_rn(acc, bilinear_rn(t, Ia, Ib, Ic, Id));            // then reduce_mean over C (homography_model.py:263)
  }
  return C == 1 ? acc : acc / (float)C;
}

// d gray / dx and d gray / dy through the weights only (floor/clip/gather are not differentiable).
template <int C>
__device__ __forceinline__ void sample_grad(const float* __restrict__ img, const Tap& t, float& gx, float& gy) {
  float ax = 0.f, ay = 0.f;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const float Ia = __ldg(img + (size_t)t.i00 * C + c), Ib = __ldg(img + (size_t)t.i10 * C + c);
    const float Ic = __ldg(img + (size_t)t.i01 * C + c), Id = __ldg(img + (size_t)t.i11 * C + c);
    ax += (t.y1f - t.y) * (Ic - Ia) + (t.y - t.y0f) * (Id - Ib);
    ay += (t.x1f - t.x) * (Ib - Ia) + (t.x - t.x0f) * (Id - Ic);
  }
  gx = C == 1 ? ax : ax / (float)C;
  gy = C == 1 ? ay : ay / (float)C;
}

__device__ __forceinline__ void window_origin(const int32_t* __restrict__ patch_indices, int64_t idx_stride, int b,
                                              int img_w, int& ox, int& oy) {
  ox = 0; oy = 0;
  if (patch_indices) {
    const int idx0 = __ldg(patch_indices + (size_t)b * idx_stride);   // (y0)*W + x0, dataloader.py:203-207
    oy = idx0 / img_w; ox = idx0 - oy * img_w;
  }
}

// ------------------------------------------------------------------------------------------------------------
// forward: grid (X, B), 256 threads.  A sample's window is a flat list of ph * pw/4 pixel quads (4 consecutive pixels of a
// row); thread t of CTA x takes quads x*256 + t, + X*256, ...: every warp reads / writes 512 contiguous bytes of I2 / pred
// per iteration whatever the window width (a 320-wide row is 2.5 warps, no idle lanes), and X is chosen so that B * X CTAs
// fill the device once (no second, mostly empty wave).
// In-range samples (the common case) take a fast path; samples whose taps clip go through the general clip-then-weight
// path.  The choice is made PER WARP AND QUAD (__all_sync): a warp that straddles the image border runs the general path for
// all of its lanes instead of both paths one after the other — the two produce the same fp32 weights for in-range samples.
// Reductions: fp32 over the thread's pixels, then fp64.
// ------------------------------------------------------------------------------------------------------------
// Source position (pixels) of the output grid point with abscissa xt on a row whose constant terms are (bx, by, bt).
__device__ __forceinline__ void source_xy(const Homog& hm, float xt, float bx, float by, float bt, int W, int Hh, float& x, float& y) {
  const float xs = fmaf(hm.h[0], xt, bx), ys = fmaf(hm.h[3], xt, by);
  float ts = fmaf(hm.h[6], xt, bt);
  if (!(fabsf(ts) >= 1e-7f)) ts += 1e-6f;
  // ONE hardware reciprocal (MUFU.RCP, <= 1 ulp) instead of two IEEE divisions (the kernel is issue / latency bound, not DRAM
  // bound; a correctly rounded __frcp_rn costs ~8 instructions, this one 1): xs * (1/ts) is within 2 ulp of xs / ts,
  // i.e. < 7e-5 px on coordinates of a few hundred px — far inside the parity tolerance of the warp (2e-4 on 99.9 % of the
  // pixels).  |ts| >= 1e-7 here (epsilon rule above), so the .ftz of the approximation never sees a denormal.
  float rt;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rt) : "f"(ts));
  x = (xs * rt + 1.0f) * (float)W * 0.5f;
  y = (ys * rt + 1.0f) * (float)Hh * 0.5f;
}

// The four pixels of a quad.  Fast path (no tap of any pixel of the WARP clips: floor == truncation, x1 = x0 + 1 — the same
// fp32 weights as the general path): all 16 C texel loads of the quad are issued before the first blend.
template <int C>
__device__ __forceinline__ void sample_quad(const float* __restrict__ img, const Homog& hm, const float (&xt)[4], float bx, float by,
                                            float bt, int W, int Hh, float (&out)[4]) {
  float x[4], y[4];
  bool inside = true;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    source_xy(hm, xt[k], bx, by, bt, W, Hh, x[k], y[k]);
    inside = inside && x[k] >= 0.0f && x[k] < (float)(W - 1) && y[k] >= 0.0f && y[k] < (float)(Hh - 1);
  }
  if (__all_sync(0xffffffffu, inside)) {
    float wa[4], wb[4], wc[4], wd[4];
    const float* p0[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int x0 = (int)x[k], y0 = (int)y[k];
      const float x0f = (float)x0, y0f = (float)y0;
      const float dx1 = (x0f + 1.0f) - x[k], dx0 = x[k] - x0f, dy1 = (y0f + 1.0f) - y[k], dy0 = y[k] - y0f;
      wa[k] = __fmul_rn(dx1, dy1); wb[k] = __fmul_rn(dx1, dy0); wc[k] = __fmul_rn(dx0, dy1); wd[k] = __fmul_rn(dx0, dy0);
      p0[k] = img + (y0 * W + x0) * C;
    }
    if (C == 1) {
      float Ia[4], Ib[4], Ic[4], Id[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        Ia[k] = __ldg(p0[k]); Ic[k] = __ldg(p0[k] + 1); Ib[k] = __ldg(p0[k] + W); Id[k] = __ldg(p0[k] + W + 1);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k)
        out[k] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(wa[k], Ia[k]), __fmul_rn(wb[k], Ib[k])), __fmul_rn(wc[k], Ic[k])), __fmul_rn(wd[k], Id[k]));
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float* p1 = p0[k] + W * C;
        float acc = 0.f;
#pragma unroll
        for (int c = 0; c < C; ++c) {
          const float Ia = __ldg(p0[k] + c), Ic = __ldg(p0[k] + C + c), Ib = __ldg(p1 + c), Id = __ldg(p1 + C + c);
          acc = __fadd_rn(acc, __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(wa[k], Ia), __fmul_rn(wb[k], Ib)), __fmul_rn(wc[k], Ic)), __fmul_rn(wd[k], Id)));
        }
        out[k] = acc / (float)C;
      }
    }
    return;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    Tap t;
    tap_from_xy(x[k], y[k], W, Hh, t);
    out[k] = sample_gray<C>(img, t);
  }
}

// ALL = true: the six reductions every photometric diagnostic needs; false: sum |pred - I2| only (l1_loss)
template <int C, bool ALL>
__global__ void __launch_bounds__(256) warp_loss_fwd_kernel(const float* __restrict__ I, int img_h, int img_w,
                                                            const float* __restrict__ H, const float* __restrict__ I2,
                                                            const int32_t* __restrict__ patch_indices, int64_t idx_stride,
                                                            int pw, int ph, float* __restrict__ pred,
                                                            double* __restrict__ sums) {
  pdl_wait(); pdl_trigger();   // launched through launch_chain (common.cuh)
  __shared__ double red[UDH_NSUMS * 32];
  __shared__ Homog hm_s;
  __shared__ int org_s[2];
  const int b = blockIdx.y;
  if (threadIdx.x == 0) {
    // per-sample constants once per CTA (their IEEE divisions are ~200 instructions; a thread only samples ~16 pixels)
    Homog h0;
    normalise_h(H + (size_t)b * 9, img_w, img_h, h0);
    h0.step_x = 2.0f / (float)(img_w - 1);                   // TF LinSpace: step = (stop-start)/(num-1)
    h0.step_y = 2.0f / (float)(img_h - 1);
    hm_s = h0;
    window_origin(patch_indices, idx_stride, b, img_w, org_s[0], org_s[1]);
  }
  __syncthreads();
  const Homog hm = hm_s;
  const int ox = org_s[0], oy = org_s[1];
  const float* img = I + (size_t)b * img_h * img_w * C;
  const int pw4 = pw >> 2, Q = ph * pw4;                     // quads per row / per sample
  const int stride = gridDim.x * 256;
  const int dr = stride / pw4, dc = stride - dr * pw4;       // the stride in (row, quad-of-row) steps
  int q = blockIdx.x * 256 + threadIdx.x;
  int r = q / pw4, cq = q - r * pw4;

  float s_abs = 0.f, s_sq = 0.f, s_hub = 0.f, s_xy = 0.f, s_xx = 0.f, s_yy = 0.f;
  // the trip count is warp-uniform (sample_quad votes across the warp): lanes past the end recompute the last quad, unused
  for (int q0 = q - (int)(threadIdx.x & 31); q0 < Q; q0 += stride) {
    const bool live = q < Q;
    const int rr = live ? r : ph - 1, c0 = (live ? cq : pw4 - 1) << 2;
    const float yt = fmaf(hm.step_y, (float)(oy + rr), -1.0f);
    // row-constant parts of T_g = H' . (x_t, y_t, 1): identical to fmaf(h0, xt, fmaf(h1, yt, h2)) etc.
    const float bx = fmaf(hm.h[1], yt, hm.h[2]), by = fmaf(hm.h[4], yt, hm.h[5]), bt = fmaf(hm.h[7], yt, hm.h[8]);
    float p[4], xt[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) xt[k] = fmaf(hm.step_x, (float)(ox + c0 + k), -1.0f);
    sample_quad<C>(img, hm, xt, bx, by, bt, img_w, img_h, p);
    if (live) {
      const size_t o = ((size_t)b * ph + rr) * pw + c0;
      if (pred) *reinterpret_cast<float4*>(pred + o) = make_float4(p[0], p[1], p[2], p[3]);
      if (I2) {
        const float4 tv = __ldg(reinterpret_cast<const float4*>(I2 + o));
        const float tg[4] = {tv.x, tv.y, tv.z, tv.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float d = p[k] - tg[k], ad = fabsf(d);
          s_abs += ad;
          if (ALL) {
            s_sq = fmaf(d, d, s_sq);
            s_hub += ad < 1.0f ? 0.5f * d * d : ad - 0.5f;
            s_xy = fmaf(p[k], tg[k], s_xy);
            s_xx = fmaf(p[k], p[k], s_xx);
            s_yy = fmaf(tg[k], tg[k], s_yy);
          }
        }
      }
    }
    q += stride; r += dr; cq += dc;
    if (cq >= pw4) { cq -= pw4; ++r; }
  }
  if (sums && I2) {
    if (ALL) {
      double acc[6] = {s_abs, s_sq, s_hub, s_xy, s_xx, s_yy};
      block_sum<double, 6>(acc, red);
      if (threadIdx.x == 0) {
#pragma unroll
        for (int i = 0; i < 6; ++i) atomicAdd(sums + i, acc[i]);
      }
    } else {
      double acc[1] = {s_abs};
      block_sum<double, 1>(acc, red);
      if (threadIdx.x == 0) atomicAdd(sums + UDH_SUM_ABS, acc[0]);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// backward: d loss / d H' accumulated per sample with block reductions + 9 float atomics per CTA.
// ------------------------------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(256) warp_loss_bwd_kernel(const float* __restrict__ I, int img_h, int img_w,
                                                            const float* __restrict__ H, const float* __restrict__ I2,
                                                            const int32_t* __restrict__ patch_indices, int64_t idx_stride,
                                                            int pw, int ph, int loss_type, const double* __restrict__ sums,
                                                            const float* __restrict__ dpred, float upstream, double n_total,
                                                            float* __restrict__ dHn) {
  __shared__ float red[9 * 32];
  const int b = blockIdx.y;
  const int tiles_x = (pw + 127) >> 7;
  const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x;
  const int c0 = (tx << 7) + ((threadIdx.x & 31) << 2);
  const int r = (ty << 3) + (threadIdx.x >> 5);
  Homog hm;
  normalise_h(H + (size_t)b * 9, img_w, img_h, hm);
  hm.step_x = 2.0f / (float)(img_w - 1);
  hm.step_y = 2.0f / (float)(img_h - 1);
  int ox, oy;
  window_origin(patch_indices, idx_stride, b, img_w, ox, oy);
  const float* img = I + (size_t)b * img_h * img_w * C;

  // d loss / d pred = coef * f(d):  L1: sign(d)/N;  REC: d/(N*rec);  L1_SMOOTH: clamp(d,-1,1)/N
  //   NCC (homography_model.py:161-166): ncc = sqrt(2 - 2c), c = <p,t>/(|p||t|):  d ncc/d p_i = -(t_i/(|p||t|) - c p_i/|p|^2)/ncc
  //   CUSTOM: d loss / d pred is given per pixel (used for ssim_loss, whose 3x3 windows couple neighbouring pixels)
  float coef = upstream / (float)n_total;
  float ncc_a = 0.f, ncc_b = 0.f;
  if (loss_type == UDH_LOSS_REC) coef = upstream / (float)(n_total * sqrt(sums[UDH_SUM_SQ] / n_total));
  if (loss_type == UDH_LOSS_NCC) {
    const double pp = sums[UDH_SUM_XX], tt = sums[UDH_SUM_YY], c = sums[UDH_SUM_XY] / sqrt(pp * tt);
    const double ncc = sqrt(fmax(1e-30, 2.0 - 2.0 * c));
    ncc_a = (float)(-(double)upstream / (ncc * sqrt(pp * tt)));
    ncc_b = (float)((double)upstream * c / (ncc * pp));
  }

  float g[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  if (r < ph && c0 < pw) {
    const float yt = fmaf(hm.step_y, (float)(oy + r), -1.0f);
    const size_t o = ((size_t)b * ph + r) * pw + c0;
    const float4 tv = __ldg(reinterpret_cast<const float4*>(I2 + o));
    const float tg[4] = {tv.x, tv.y, tv.z, tv.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float xt = fmaf(hm.step_x, (float)(ox + c0 + k), -1.0f);
      Tap t;
      sample_setup(hm, xt, yt, img_w, img_h, t);
      const float pv = sample_gray<C>(img, t);
      const float d = pv - tg[k];
      float gp;
      if (loss_type == UDH_LOSS_L1) gp = (d > 0.f) ? coef : ((d < 0.f) ? -coef : 0.f);
      else if (loss_type == UDH_LOSS_REC) gp = coef * d;
      else if (loss_type == UDH_LOSS_L1_SMOOTH) gp = coef * fminf(fmaxf(d, -1.0f), 1.0f);
      else if (loss_type == UDH_LOSS_NCC) gp = fmaf(ncc_a, tg[k], ncc_b * pv);
      else gp = upstream * __ldg(dpred + o + k);
      float gx, gy;
      sample_grad<C>(img, t, gx, gy);
      const float Gx = gp * gx * (0.5f * (float)img_w);      // through x = (xn+1)*W/2
      const float Gy = gp * gy * (0.5f * (float)img_h);
      const float inv_t = 1.0f / t.ts;
      const float dxs = Gx * inv_t, dys = Gy * inv_t;
      const float dts = -(Gx * t.xn + Gy * t.yn) * inv_t;
      g[0] = fmaf(dxs, xt, g[0]); g[1] = fmaf(dxs, yt, g[1]); g[2] += dxs;
      g[3] = fmaf(dys, xt, g[3]); g[4] = fmaf(dys, yt, g[4]); g[5] += dys;
      g[6] = fmaf(dts, xt, g[6]); g[7] = fmaf(dts, yt, g[7]); g[8] += dts;
    }
  }
  block_sum<float, 9>(g, red);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < 9; ++i) atomicAdd(dHn + (size_t)b * 9 + i, g[i]);
  }
}

// dH = Minv^T . dH' . M^T  (adjoint of H' = Minv . H . M)
__global__ void conj_bwd_kernel(const float* __restrict__ dHn, float* __restrict__ dH, int img_w, int img_h, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float sx = 0.5f * (float)img_w, sy = 0.5f * (float)img_h;
  const float ix = 1.0f / sx, iy = 1.0f / sy;
  float g[9], t[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) g[i] = dHn[(size_t)b * 9 + i];
  // t = g . M^T : t[r][0] = sx*g[r][0] + sx*g[r][2]; t[r][1] = sy*g[r][1] + sy*g[r][2]; t[r][2] = g[r][2]
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    t[3 * r + 0] = sx * (g[3 * r + 0] + g[3 * r + 2]);
    t[3 * r + 1] = sy * (g[3 * r + 1] + g[3 * r + 2]);
    t[3 * r + 2] = g[3 * r + 2];
  }
  // dH = Minv^T . t, Minv^T = [[ix,0,0],[0,iy,0],[-1,-1,1]]
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    dH[(size_t)b * 9 + c] = ix * t[c];
    dH[(size_t)b * 9 + 3 + c] = iy * t[3 + c];
    dH[(size_t)b * 9 + 6 + c] = t[6 + c] - t[c] - t[3 + c];
  }
}

// ------------------------------------------------------------------------------------------------------------
// SSIM diagnostic (homography_model.py:141-158): 3x3 VALID average pools of x, y, x^2, y^2, xy.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ssim_kernel(const float* __restrict__ X, const float* __restrict__ Y, int pw, int ph,
                                                   double* __restrict__ sums) {
  pdl_wait(); pdl_trigger();   // launched through launch_chain (common.cuh)
  __shared__ double red[32];
  const int b = blockIdx.y;
  const int ow = pw - 2, oh = ph - 2;
  const float* x = X + (size_t)b * pw * ph;
  const float* y = Y + (size_t)b * pw * ph;
  double acc[1] = {0.0};
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < ow * oh; o += gridDim.x * blockDim.x) {
    const int r = o / ow, c = o - r * ow;
    float sx = 0, sy = 0, sxx = 0, syy = 0, sxy = 0;
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        const float a = __ldg(x + (r + dy) * pw + c + dx), bb = __ldg(y + (r + dy) * pw + c + dx);
        sx += a; sy += bb; sxx = fmaf(a, a, sxx); syy = fmaf(bb, bb, syy); sxy = fmaf(a, bb, sxy);
      }
    const float k = 1.0f / 9.0f;
    const float mu_x = sx * k, mu_y = sy * k;
    const float sig_x = sxx * k - mu_x * mu_x, sig_y = syy * k - mu_y * mu_y, sig_xy = sxy * k - mu_x * mu_y;
    const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
    const float n = (2.f * mu_x * mu_y + C1) * (2.f * sig_xy + C2);
    const float d = (mu_x * mu_x + mu_y * mu_y + C1) * (sig_x + sig_y + C2);
    acc[0] += (double)fminf(fmaxf((1.0f - n / d) * 0.5f, 0.f), 1.f);
  }
  block_sum<double, 1>(acc, red);
  if (threadIdx.x == 0) atomicAdd(sums + UDH_SUM_SSIM, acc[0]);
}

// d mean(clip((1-SSIM)/2,0,1)) / d pred, one thread per pixel: every 3x3 window containing the pixel is re-evaluated.
__global__ void __launch_bounds__(256) ssim_bwd_kernel(const float* __restrict__ X, const float* __restrict__ Y, int pw, int ph,
                                                       float inv_n, float* __restrict__ dX) {
  const int b = blockIdx.y;
  const float* x = X + (size_t)b * pw * ph;
  const float* y = Y + (size_t)b * pw * ph;
  const int ow = pw - 2, oh = ph - 2;
  const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f, k = 1.0f / 9.0f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < pw * ph; i += gridDim.x * blockDim.x) {
    const int r = i / pw, c = i - r * pw;
    const float xi = x[i], yi = y[i];
    float g = 0.f;
    for (int wy = max(0, r - 2); wy <= min(oh - 1, r); ++wy)
      for (int wx = max(0, c - 2); wx <= min(ow - 1, c); ++wx) {
        float sx = 0, sy = 0, sxx = 0, syy = 0, sxy = 0;
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
          for (int dx = 0; dx < 3; ++dx) {
            const float a = __ldg(x + (wy + dy) * pw + wx + dx), bb = __ldg(y + (wy + dy) * pw + wx + dx);
            sx += a; sy += bb; sxx = fmaf(a, a, sxx); syy = fmaf(bb, bb, syy); sxy = fmaf(a, bb, sxy);
          }
        const float mu_x = sx * k, mu_y = sy * k;
        const float sig_x = sxx * k - mu_x * mu_x, sig_y = syy * k - mu_y * mu_y, sig_xy = sxy * k - mu_x * mu_y;
        const float A1 = 2.f * mu_x * mu_y + C1, A2 = 2.f * sig_xy + C2, B1 = mu_x * mu_x + mu_y * mu_y + C1, B2 = sig_x + sig_y + C2;
        const float S = (A1 * A2) / (B1 * B2);
        const float L = (1.0f - S) * 0.5f;
        if (L > 0.f && L < 1.f) {                             // inside the clip: dL/dS = -1/2
          const float dA1 = 2.f * mu_y * k, dA2 = 2.f * (yi - mu_y) * k, dB1 = 2.f * mu_x * k, dB2 = 2.f * (xi - mu_x) * k;
          const float dS = (dA1 * A2 + A1 * dA2) / (B1 * B2) - S * (dB1 * B2 + B1 * dB2) / (B1 * B2);
          g += -0.5f * dS;
        }
      }
    dX[(size_t)b * pw * ph + i] = g * inv_n;
  }
}

__global__ void photo_finalize_kernel(const double* __restrict__ sums, double n, double n_ssim, float* __restrict__ out) {
  pdl_wait(); pdl_trigger();   // launched through launch_chain (common.cuh)
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  out[UDH_L_REC] = (float)sqrt(sums[UDH_SUM_SQ] / n);
  out[UDH_L_SSIM] = n_ssim > 0 ? (float)(sums[UDH_SUM_SSIM] / n_ssim) : 0.f;
  out[UDH_L_L1] = (float)(sums[UDH_SUM_ABS] / n);
  out[UDH_L_L1_SMOOTH] = (float)(sums[UDH_SUM_HUBER] / n);
  // ncc = || y/|y| - x/|x| ||_2 = sqrt(2 - 2 <x,y>/(|x||y|))   (homography_model.py:161-166)
  const double c = sums[UDH_SUM_XY] / sqrt(sums[UDH_SUM_XX] * sums[UDH_SUM_YY]);
  out[UDH_L_NCC] = (float)sqrt(fmax(0.0, 2.0 - 2.0 * c));
  out[5] = 0.f; out[6] = 0.f; out[7] = 0.f;
}

// ------------------------------------------------------------------------------------------------------------
// the `transformer` operator: full output grid, all channels, theta already normalised.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) transformer_kernel(const float* __restrict__ U, const float* __restrict__ theta,
                                                          float* __restrict__ out, int H, int W, int C, int oh, int ow) {
  const int b = blockIdx.y;
  Homog hm;
#pragma unroll
  for (int i = 0; i < 9; ++i) hm.h[i] = theta[(size_t)b * 9 + i];
  hm.step_x = 2.0f / (float)(ow - 1);
  hm.step_y = 2.0f / (float)(oh - 1);
  const float* img = U + (size_t)b * H * W * C;
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < oh * ow; o += gridDim.x * blockDim.x) {
    const int r = o / ow, c = o - r * ow;
    Tap t;
    sample_setup(hm, fmaf(hm.step_x, (float)c, -1.0f), fmaf(hm.step_y, (float)r, -1.0f), W, H, t);
    float* dst = out + ((size_t)b * oh * ow + o) * C;
    for (int ch = 0; ch < C; ++ch) {
      const float Ia = __ldg(img + (size_t)t.i00 * C + ch), Ib = __ldg(img + (size_t)t.i10 * C + ch);
      const float Ic = __ldg(img + (size_t)t.i01 * C + ch), Id = __ldg(img + (size_t)t.i11 * C + ch);
      dst[ch] = bilinear_rn(t, Ia, Ib, Ic, Id);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// synthetic-pair generation (code/utils/gen_synthetic_data.py:56-64): I' = warp of the uint8 image I with the pixel-unit
// homography H (theta = M^-1 H M, numpy_spatial_transformer.py:135-146), cast back to uint8 (:131).  Same sampling code as
// the training-time warp above, uint8 in / uint8 out, all 3 channels of a pixel per thread.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) warp_image_u8_kernel(const uint8_t* __restrict__ U, const float* __restrict__ H,
                                                            uint8_t* __restrict__ out, int Hh, int W) {
  const int b = blockIdx.y;
  Homog hm;
  normalise_h(H + (size_t)b * 9, W, Hh, hm);
  hm.step_x = 2.0f / (float)(W - 1);
  hm.step_y = 2.0f / (float)(Hh - 1);
  const uint8_t* img = U + (size_t)b * Hh * W * 3;
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < Hh * W; o += gridDim.x * blockDim.x) {
    const int r = o / W, c = o - r * W;
    Tap t;
    sample_setup(hm, fmaf(hm.step_x, (float)c, -1.0f), fmaf(hm.step_y, (float)r, -1.0f), W, Hh, t);
    uint8_t* dst = out + ((size_t)b * Hh * W + o) * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float Ia = (float)__ldg(img + (size_t)t.i00 * 3 + ch), Ib = (float)__ldg(img + (size_t)t.i10 * 3 + ch);
      const float Ic = (float)__ldg(img + (size_t)t.i01 * 3 + ch), Id = (float)__ldg(img + (size_t)t.i11 * 3 + ch);
      const float v = bilinear_rn(t, Ia, Ib, Ic, Id);
      dst[ch] = (uint8_t)fminf(fmaxf(v, 0.0f), 255.0f);       // clamp, then truncate like astype(uint8)
    }
  }
}

}  // namespace udh

using namespace udh;

extern "C" int udh_warp_image_u8(const uint8_t* U, const float* H, uint8_t* out, int B, int img_h, int img_w, void* stream) {
  UDH_REQUIRE(U && H && out, "udh_warp_image_u8: null pointer");
  UDH_REQUIRE(B >= 0 && img_h >= 2 && img_w >= 2, "udh_warp_image_u8: bad dimensions");
  if (B == 0) return UDH_OK;
  dim3 grid(min((img_h * img_w + 255) / 256, 1024), B);
  warp_image_u8_kernel<<<grid, 256, 0, as_stream(stream)>>>(U, H, out, img_h, img_w);
  return check_launch("udh_warp_image_u8");
}

static int check_warp_args(const char* fn, const float* I, int C, int img_h, int img_w, const float* H, int pw, int ph,
                           int B) {
  UDH_REQUIRE(I && H, "%s: null image or homography pointer", fn);
  UDH_REQUIRE(C == 1 || C == 3, "%s: C must be 1 or 3 (got %d)", fn, C);
  UDH_REQUIRE(img_h >= 2 && img_w >= 2 && pw > 0 && ph > 0 && B >= 0, "%s: bad dimensions", fn);
  UDH_REQUIRE(pw % 4 == 0, "%s: window width must be a multiple of 4 (got %d)", fn, pw);
  return UDH_OK;
}

extern "C" int udh_warp_loss_fwd(const float* I, int C, int img_h, int img_w, const float* H, const float* I2,
                                 const int32_t* patch_indices, int64_t idx_stride, int pw, int ph, float* pred,
                                 double* sums, int B, void* stream) {
  return udh_warp_loss_fwd_ex(I, C, img_h, img_w, H, I2, patch_indices, idx_stride, pw, ph, pred, sums, 1, B, stream);
}

extern "C" int udh_warp_loss_fwd_ex(const float* I, int C, int img_h, int img_w, const float* H, const float* I2,
                                    const int32_t* patch_indices, int64_t idx_stride, int pw, int ph, float* pred,
                                    double* sums, int all_sums, int B, void* stream) {
  int rc = check_warp_args("udh_warp_loss_fwd", I, C, img_h, img_w, H, pw, ph, B);
  if (rc) return rc;
  UDH_REQUIRE(pred || (I2 && sums), "udh_warp_loss_fwd: nothing to compute (no pred, no I2+sums)");
  if (B == 0) return UDH_OK;
  // B * X CTAs of 256 threads: one full wave of the device (as many CTAs per SM as the kernel's registers allow) when the work
  // allows, never more CTAs than quads
  const int quads = ph * (pw / 4), full = (quads + 255) / 256;
  int dev = 0, sms = 148;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const void* fn = C == 3 ? (all_sums ? (const void*)warp_loss_fwd_kernel<3, true> : (const void*)warp_loss_fwd_kernel<3, false>)
                          : (all_sums ? (const void*)warp_loss_fwd_kernel<1, true> : (const void*)warp_loss_fwd_kernel<1, false>);
  int per_sm = 4;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, 256, 0) != cudaSuccess || per_sm < 1) { cudaGetLastError(); per_sm = 4; }
  int X = (sms * per_sm) / B;
  X = X < 1 ? 1 : (X > full ? full : X);
  dim3 grid(X, B);
  ProfScope ps(PROF_WARP_FWD, as_stream(stream));
  if (C == 3 && all_sums)
    launch_chain(warp_loss_fwd_kernel<3, true>, grid, dim3(256), 0, as_stream(stream), I, img_h, img_w, H, I2, patch_indices, idx_stride, pw, ph, pred, sums);
  else if (C == 3)
    launch_chain(warp_loss_fwd_kernel<3, false>, grid, dim3(256), 0, as_stream(stream), I, img_h, img_w, H, I2, patch_indices, idx_stride, pw, ph, pred, sums);
  else if (all_sums)
    launch_chain(warp_loss_fwd_kernel<1, true>, grid, dim3(256), 0, as_stream(stream), I, img_h, img_w, H, I2, patch_indices, idx_stride, pw, ph, pred, sums);
  else
    launch_chain(warp_loss_fwd_kernel<1, false>, grid, dim3(256), 0, as_stream(stream), I, img_h, img_w, H, I2, patch_indices, idx_stride, pw, ph, pred, sums);
  return check_launch("udh_warp_loss_fwd");
}

extern "C" int udh_warp_loss_bwd(const float* I, int C, int img_h, int img_w, const float* H, const float* I2,
                                 const int32_t* patch_indices, int64_t idx_stride, int pw, int ph, int loss_type,
                                 const double* sums, float upstream, float* dH, float* scratch, int B, void* stream) {
  int rc = check_warp_args("udh_warp_loss_bwd", I, C, img_h, img_w, H, pw, ph, B);
  if (rc) return rc;
  UDH_REQUIRE(I2 && dH && scratch, "udh_warp_loss_bwd: null pointer");
  return udh_warp_loss_bwd_ex(I, C, img_h, img_w, H, I2, patch_indices, idx_stride, pw, ph, loss_type, sums, nullptr, upstream, dH, scratch,
                              B, stream);
}

extern "C" int udh_warp_loss_bwd_ex(const float* I, int C, int img_h, int img_w, const float* H, const float* I2,
                                    const int32_t* patch_indices, int64_t idx_stride, int pw, int ph, int loss_type,
                                    const double* sums, const float* dpred, float upstream, float* dH, float* scratch, int B,
                                    void* stream) {
  int rc = check_warp_args("udh_warp_loss_bwd", I, C, img_h, img_w, H, pw, ph, B);
  if (rc) return rc;
  UDH_REQUIRE(I2 && dH && scratch, "udh_warp_loss_bwd: null pointer");
  UDH_REQUIRE(loss_type >= UDH_LOSS_L1 && loss_type <= UDH_LOSS_CUSTOM, "udh_warp_loss_bwd: unsupported loss_type %d", loss_type);
  UDH_REQUIRE((loss_type != UDH_LOSS_REC && loss_type != UDH_LOSS_NCC) || sums, "udh_warp_loss_bwd: REC / NCC need the forward sums");
  UDH_REQUIRE(loss_type != UDH_LOSS_CUSTOM || dpred, "udh_warp_loss_bwd: CUSTOM needs the per-pixel d loss / d pred");
  if (B == 0) return UDH_OK;
  cudaStream_t st = as_stream(stream);
  ProfScope ps(PROF_WARP_BWD, st);
  UDH_CUDA(cudaMemsetAsync(scratch, 0, sizeof(float) * 9 * (size_t)B, st));
  dim3 grid(((pw + 127) / 128) * ((ph + 7) / 8), B);
  const double n_total = (double)B * pw * ph;
  if (C == 3)
    warp_loss_bwd_kernel<3><<<grid, 256, 0, st>>>(I, img_h, img_w, H, I2, patch_indices, idx_stride, pw, ph, loss_type, sums, dpred, upstream, n_total, scratch);
  else
    warp_loss_bwd_kernel<1><<<grid, 256, 0, st>>>(I, img_h, img_w, H, I2, patch_indices, idx_stride, pw, ph, loss_type, sums, dpred, upstream, n_total, scratch);
  rc = check_launch("udh_warp_loss_bwd");
  if (rc) return rc;
  conj_bwd_kernel<<<(B + 127) / 128, 128, 0, st>>>(scratch, dH, img_w, img_h, B);
  return check_launch("udh_warp_loss_bwd(conj)");
}

extern "C" int udh_ssim_fwd(const float* pred, const float* I2, int pw, int ph, double* sums, int B, void* stream) {
  UDH_REQUIRE(pred && I2 && sums, "udh_ssim_fwd: null pointer");
  UDH_REQUIRE(pw >= 3 && ph >= 3 && B >= 0, "udh_ssim_fwd: bad dimensions");
  if (B == 0) return UDH_OK;
  const int n = (pw - 2) * (ph - 2);
  dim3 grid(min((n + 255) / 256, 64), B);
  ProfScope ps(PROF_SSIM, as_stream(stream));
  launch_chain(ssim_kernel, grid, dim3(256), 0, as_stream(stream), pred, I2, pw, ph, sums);
  return check_launch("udh_ssim_fwd");
}

extern "C" int udh_ssim_bwd(const float* pred, const float* I2, int pw, int ph, float* dpred, int B, void* stream) {
  UDH_REQUIRE(pred && I2 && dpred, "udh_ssim_bwd: null pointer");
  UDH_REQUIRE(pw >= 3 && ph >= 3 && B >= 0, "udh_ssim_bwd: bad dimensions");
  if (B == 0) return UDH_OK;
  ProfScope ps(PROF_SSIM, as_stream(stream));
  const float inv_n = 1.0f / ((float)B * (float)(pw - 2) * (float)(ph - 2));
  dim3 grid(min((pw * ph + 255) / 256, 64), B);
  ssim_bwd_kernel<<<grid, 256, 0, as_stream(stream)>>>(pred, I2, pw, ph, inv_n, dpred);
  return check_launch("udh_ssim_bwd");
}

extern "C" int udh_photo_losses_finalize(const double* sums, double n, double n_ssim, float* losses, void* stream) {
  UDH_REQUIRE(sums && losses && n > 0, "udh_photo_losses_finalize: bad arguments");
  launch_chain(photo_finalize_kernel, dim3(1), dim3(32), 0, as_stream(stream), sums, n, n_ssim, losses);
  return check_launch("udh_photo_losses_finalize");
}

extern "C" int udh_transformer_fwd(const float* U, const float* theta, float* out, int B, int H, int W, int C,
                                   int out_h, int out_w, void* stream) {
  UDH_REQUIRE(U && theta && out, "udh_transformer_fwd: null pointer");
  UDH_REQUIRE(B >= 0 && H >= 1 && W >= 1 && C >= 1 && out_h >= 2 && out_w >= 2, "udh_transformer_fwd: bad dimensions");
  if (B == 0) return UDH_OK;
  dim3 grid(min((out_h * out_w + 255) / 256, 1024), B);
  transformer_kernel<<<grid, 256, 0, as_stream(stream)>>>(U, theta, out, H, W, C, out_h, out_w);
  return check_launch("udh_transformer_fwd");
}
