// Device-side synthetic pair generation and fused input preparation (SURVEY §8f item 1), so that the input side keeps up
// with a train step of a few milliseconds:
//   udh_synth_scene_u8      seeded multi-octave texture I (uint8 NHWC) + random patch corners pts1 and corner
//                           perturbations gt drawn like code/utils/gen_synthetic_data.py:40-53
//   (udh_dlt_fwd + udh_warp_image_u8 then give H_gt and I' exactly as :56-64 do)
//   udh_prep_inputs_u8_ex   everything the reference Dataloader does after JPEG decode, in one pass over the two uint8 images
//                           (code/dataloader.py:163-177,203-227,323-375): photometric augmentation (gamma on the RAW 0..255
//                           values, brightness, per-channel colour, clip), normalisation with I's statistics, gray = channel
//                           mean, gather of the two patches — through per-sample 256-entry lookup tables per channel, since
//                           the whole per-pixel transform is a function of one uint8 value.
#include "common.cuh"

namespace udh {

__constant__ float kGenMean[3] = {118.93f, 113.97f, 102.60f};
__constant__ float kGenStd[3] = {69.85f, 68.81f, 72.45f};

__device__ __forceinline__ uint64_t mix64(uint64_t x) {                 // splitmix64: the golden-ratio step and the finaliser
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__device__ __forceinline__ uint32_t hash_u32(uint64_t x) { return (uint32_t)(mix64(x) >> 32); }
__device__ __forceinline__ float hash_unit(uint64_t key) { return (float)(hash_u32(key) >> 8) * (1.0f / 16777216.0f) - 0.5f; }   // [-0.5, 0.5)

// Key of one random stream of sample b: the seed, then b, then the stream's tag each pass through the finaliser before the
// next is mixed in, so that seeds, samples and streams that differ in a few low bits (the dataloader's seed + step,
// consecutive samples, consecutive draws) give unrelated keys.  Keying on seed ^ index or seed + index would not: a
// seed one apart then shifts or permutes the other seed's draws.  Tags: 3 * 6 texture lattices (c * 6 + o), then the
// corner draws.
__device__ __forceinline__ uint64_t stream_key(uint64_t seed, int b, int tag) {
  return mix64(mix64(mix64(seed) ^ (uint64_t)(uint32_t)b) ^ (uint64_t)(uint32_t)tag);
}
constexpr int kTagCorners = 18;

// lattice value at integer (gx, gy) of the lattice whose stream key is k (one per sample, channel and octave)
__device__ __forceinline__ float lattice(uint64_t k, int gx, int gy) {
  return hash_unit(k ^ ((uint64_t)(uint32_t)gx | ((uint64_t)(uint32_t)gy << 32)));
}

// Multi-octave value noise: lattices at 1, 1/2, ... 1/32 resolution, smoothstep-interpolated, amplitude 2^(0.9 o)
// (roughly the 1/f spectrum of natural images: structure at the scale of the rho = 45 px displacements and fine detail).
__global__ void __launch_bounds__(256) texture_u8_kernel(uint8_t* __restrict__ out, int Hh, int W, uint64_t seed) {
  const int b = blockIdx.y;
  __shared__ uint64_t key[3][6];
  if (threadIdx.x < 18) key[threadIdx.x / 6][threadIdx.x % 6] = stream_key(seed, b, threadIdx.x);
  __syncthreads();
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < Hh * W; o += gridDim.x * blockDim.x) {
    const int y = o / W, x = o - y * W;
    uint8_t* dst = out + ((size_t)b * Hh * W + o) * 3;
#pragma unroll 1
    for (int c = 0; c < 3; ++c) {
      float v = lattice(key[c][0], x, y);
      float amp = 1.0f;
#pragma unroll
      for (int oc = 1; oc < 6; ++oc) {
        amp *= 1.8660660f;                                                // 2^0.9
        const float fx = (float)x / (float)(1 << oc), fy = (float)y / (float)(1 << oc);
        const int gx = (int)fx, gy = (int)fy;
        float tx = fx - (float)gx, ty = fy - (float)gy;
        tx = tx * tx * (3.0f - 2.0f * tx); ty = ty * ty * (3.0f - 2.0f * ty);
        const float a = lattice(key[c][oc], gx, gy), bb = lattice(key[c][oc], gx + 1, gy);
        const float cc = lattice(key[c][oc], gx, gy + 1), d = lattice(key[c][oc], gx + 1, gy + 1);
        v = fmaf(amp, (a + (bb - a) * tx) + ((cc + (d - cc) * tx) - (a + (bb - a) * tx)) * ty, v);
      }
      dst[c] = (uint8_t)fminf(fmaxf(127.5f + v * 9.8f, 0.0f), 255.0f);
    }
  }
}

// pts1 = (x0,y0),(x0+P,y0),(x0+P,y0+P),(x0,y0+P) with x0 in [rho, W-rho-P], y0 in [rho, Hh-rho-P]; gt integer in [-rho, rho]^8
__global__ void corners_kernel(float* __restrict__ pts1, float* __restrict__ gt, int B, int Hh, int W, int P, int rho, uint64_t seed) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  // draw i of sample b: hash_u32 of its own stream key (0: x0, 1: y0, 2..9: gt)
  const int x0 = rho + (int)(hash_u32(stream_key(seed, b, kTagCorners)) % (uint32_t)(W - 2 * rho - P + 1));
  const int y0 = rho + (int)(hash_u32(stream_key(seed, b, kTagCorners + 1)) % (uint32_t)(Hh - 2 * rho - P + 1));
  const float xs[4] = {(float)x0, (float)(x0 + P), (float)(x0 + P), (float)x0};
  const float ys[4] = {(float)y0, (float)y0, (float)(y0 + P), (float)(y0 + P)};
#pragma unroll
  for (int i = 0; i < 4; ++i) { pts1[b * 8 + 2 * i] = xs[i]; pts1[b * 8 + 2 * i + 1] = ys[i]; }
#pragma unroll
  for (int i = 0; i < 8; ++i) gt[b * 8 + i] = (float)((int)(hash_u32(stream_key(seed, b, kTagCorners + 2 + i)) % (uint32_t)(2 * rho + 1)) - rho);
}

// ---- fused augment + normalise + gray + patch gather ---------------------------------------------------------------
// aug: [B][11] = {on, gamma_I, bright_I, colR_I, colG_I, colB_I, gamma_Ip, bright_Ip, colR_Ip, colG_Ip, colB_Ip} (nullable)
__global__ void __launch_bounds__(256, 8) prep_u8_ex_kernel(const uint8_t* __restrict__ I, const uint8_t* __restrict__ Ip,
                                                         const float* __restrict__ pts1, const float* __restrict__ aug,
                                                         float* __restrict__ I_gray, float* __restrict__ I_aug3,
                                                         float* __restrict__ I1, float* __restrict__ I2, float* __restrict__ I1_aug,
                                                         float* __restrict__ I2_aug, int32_t* __restrict__ origin, int img_h, int img_w,
                                                         int P) {
  __shared__ float lut[2][3][256];
  const int b = blockIdx.y;
  const bool on = aug && aug[b * 11] != 0.0f;
  // img ** gamma on the raw 0..255 value: pow in fp64 rounded once to fp32, as denorm_u8 (common.cuh) and the ECC and
  // report tables define it, so that one augmentation row gives the same pixels on every path.  Gamma is per image, so
  // each (image, value) takes one pow for its three channels.
  for (int i = threadIdx.x; i < 2 * 256; i += blockDim.x) {
    const int im = i >> 8, x = i & 255;
    const float* a = on ? aug + b * 11 + 1 + im * 5 : nullptr;
    const float p = on ? (float)pow((double)x, (double)a[0]) : 0.0f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = (float)x;
      if (on) {
        v = __fmul_rn(p, a[1]);                                            // brightness
        v = __fmul_rn(v, a[2 + c]);                                        // colour
        v = fminf(fmaxf(v, 0.0f), 255.0f);                                 // clip_by_value(0, 255)
      }
      lut[im][c][x] = __fdiv_rn(v - kGenMean[c], kGenStd[c]);              // both images use I's statistics (dataloader.py:173-177)
    }
  }
  __syncthreads();
  const int x0 = (int)pts1[b * 8], y0 = (int)pts1[b * 8 + 1];
  if (blockIdx.x == 0 && threadIdx.x == 0 && origin) origin[b] = y0 * img_w + x0;
  const size_t img_px = (size_t)img_h * img_w;
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < img_h * img_w; o += gridDim.x * blockDim.x) {
    const int r = o / img_w, c = o - r * img_w;
    const uint8_t* p = I + ((size_t)b * img_px + o) * 3;
    const uint8_t* q = Ip + ((size_t)b * img_px + o) * 3;
    const uint8_t pr = p[0], pg = p[1], pb = p[2];
    const float ar = lut[0][0][pr], ag = lut[0][1][pg], ab = lut[0][2][pb];
    const float gI = ((ar + ag) + ab) / 3.0f;
    if (I_gray) I_gray[(size_t)b * img_px + o] = gI;
    if (I_aug3) { float* d = I_aug3 + ((size_t)b * img_px + o) * 3; d[0] = ar; d[1] = ag; d[2] = ab; }
    const int pr_ = r - y0, pc_ = c - x0;
    if (pr_ >= 0 && pr_ < P && pc_ >= 0 && pc_ < P) {
      const size_t po = ((size_t)b * P + pr_) * P + pc_;
      const uint8_t qr = q[0], qg = q[1], qb = q[2];
      I1_aug[po] = gI;
      I2_aug[po] = ((lut[1][0][qr] + lut[1][1][qg]) + lut[1][2][qb]) / 3.0f;
      if (I1) {
        I1[po] = ((__fdiv_rn((float)pr - kGenMean[0], kGenStd[0]) + __fdiv_rn((float)pg - kGenMean[1], kGenStd[1])) +
                  __fdiv_rn((float)pb - kGenMean[2], kGenStd[2])) / 3.0f;
        I2[po] = ((__fdiv_rn((float)qr - kGenMean[0], kGenStd[0]) + __fdiv_rn((float)qg - kGenMean[1], kGenStd[1])) +
                  __fdiv_rn((float)qb - kGenMean[2], kGenStd[2])) / 3.0f;
      }
    }
  }
}

}  // namespace udh

using namespace udh;

extern "C" int udh_synth_scene_u8(uint8_t* I, float* pts1, float* gt, int B, int img_h, int img_w, int P, int rho, uint64_t seed,
                                  void* stream) {
  UDH_REQUIRE(I && pts1 && gt, "udh_synth_scene_u8: null pointer");
  UDH_REQUIRE(B >= 1 && img_w - 2 * rho - P >= 0 && img_h - 2 * rho - P >= 0 && img_w < 65536 && img_h < 65536,
              "udh_synth_scene_u8: the image (%d x %d) cannot hold a %d-pixel patch with a margin of %d", img_w, img_h, P, rho);
  cudaStream_t st = as_stream(stream);
  dim3 grid(min((img_h * img_w + 255) / 256, 1024), B);
  texture_u8_kernel<<<grid, 256, 0, st>>>(I, img_h, img_w, seed);
  int rc = check_launch("texture_u8");
  if (rc) return rc;
  corners_kernel<<<(B + 127) / 128, 128, 0, st>>>(pts1, gt, B, img_h, img_w, P, rho, seed);
  return check_launch("corners");
}

extern "C" int udh_prep_inputs_u8_ex(const uint8_t* I, const uint8_t* I_prime, const float* pts1, const float* aug, float* I_gray,
                                     float* I_aug3, float* I1, float* I2, float* I1_aug, float* I2_aug, int32_t* patch_origin, int B,
                                     int img_h, int img_w, int P, void* stream) {
  UDH_REQUIRE(I && I_prime && pts1 && I1_aug && I2_aug && (I_gray || I_aug3), "udh_prep_inputs_u8_ex: null pointer");
  UDH_REQUIRE((I1 == nullptr) == (I2 == nullptr), "udh_prep_inputs_u8_ex: I1 and I2 go together");
  UDH_REQUIRE(B >= 1 && img_h >= P && img_w >= P, "udh_prep_inputs_u8_ex: bad dimensions");
  cudaStream_t st = as_stream(stream);
  ProfScope ps(PROF_ELTWISE, st);
  dim3 grid(min((img_h * img_w + 1023) / 1024, 256), B);
  prep_u8_ex_kernel<<<grid, 256, 0, st>>>(I, I_prime, pts1, aug, I_gray, I_aug3, I1, I2, I1_aug, I2_aug, patch_origin, img_h, img_w, P);
  return check_launch("udh_prep_inputs_u8_ex");
}
