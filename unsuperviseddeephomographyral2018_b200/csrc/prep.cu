// Device-side input pipeline (SURVEY §8f item 1): what the reference Dataloader does on the host after JPEG decode
// (code/dataloader.py:99-100,172-177,203-227) — normalise with I's statistics, gray = channel mean, gather the two
// 128x128 patches at (x0, y0) = pts1[0:2] — from uint8 images, so a step's host->device traffic is the decoded uint8
// images (59 MB at B = 128) instead of the fp32 post-dataloader tensors (135 MB).
#include "common.cuh"

namespace udh {

__constant__ float kMean[3] = {118.93f, 113.97f, 102.60f};
__constant__ float kStd[3] = {69.85f, 68.81f, 72.45f};

// I_aug[i] = (u8 - mean_c) / std_c over the whole image, 4 values per thread
__global__ void normalise_u8_kernel(const uint8_t* __restrict__ src, float* __restrict__ dst, size_t n4) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    const uchar4 u = __ldg(reinterpret_cast<const uchar4*>(src) + i);
    const int c0 = (int)((i * 4) % 3);
    float4 o;
    o.x = __fdiv_rn((float)u.x - kMean[c0], kStd[c0]);
    o.y = __fdiv_rn((float)u.y - kMean[(c0 + 1) % 3], kStd[(c0 + 1) % 3]);
    o.z = __fdiv_rn((float)u.z - kMean[(c0 + 2) % 3], kStd[(c0 + 2) % 3]);
    o.w = __fdiv_rn((float)u.w - kMean[c0], kStd[c0]);
    reinterpret_cast<float4*>(dst)[i] = o;
  }
}

__device__ __forceinline__ float gray_norm(const uint8_t* __restrict__ p) {
  const float a = __fdiv_rn((float)p[0] - kMean[0], kStd[0]);
  const float b = __fdiv_rn((float)p[1] - kMean[1], kStd[1]);
  const float c = __fdiv_rn((float)p[2] - kMean[2], kStd[2]);
  return ((a + b) + c) / 3.0f;
}

__global__ void patches_u8_kernel(const uint8_t* __restrict__ I, const uint8_t* __restrict__ Ip, const float* __restrict__ pts1,
                                  float* __restrict__ I1, float* __restrict__ I2, int32_t* __restrict__ origin, int img_h,
                                  int img_w, int P) {
  const int b = blockIdx.y;
  const int x0 = (int)pts1[b * 8], y0 = (int)pts1[b * 8 + 1];
  if (blockIdx.x == 0 && threadIdx.x == 0) origin[b] = y0 * img_w + x0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P * P; i += gridDim.x * blockDim.x) {
    const int r = i / P, c = i - r * P;
    const size_t src = (((size_t)b * img_h + y0 + r) * img_w + x0 + c) * 3;
    I1[(size_t)b * P * P + i] = gray_norm(I + src);
    I2[(size_t)b * P * P + i] = gray_norm(Ip + src);
  }
}

}  // namespace udh

extern "C" int udh_prep_inputs_u8(const uint8_t* I, const uint8_t* I_prime, const float* pts1, float* I_aug, float* I1, float* I2,
                                  int32_t* patch_origin, int B, int img_h, int img_w, int P, void* stream) {
  UDH_REQUIRE(I && I_prime && pts1 && I_aug && I1 && I2 && patch_origin, "udh_prep_inputs_u8: null pointer");
  UDH_REQUIRE(B >= 1 && ((size_t)B * img_h * img_w * 3) % 4 == 0, "udh_prep_inputs_u8: image bytes per batch must be a multiple of 4");
  cudaStream_t st = udh::as_stream(stream);
  udh::ProfScope ps(udh::PROF_ELTWISE, st);
  const size_t n4 = (size_t)B * img_h * img_w * 3 / 4;
  udh::normalise_u8_kernel<<<(unsigned)((n4 + 255) / 256 < udh::kSmCount * 16 ? (n4 + 255) / 256 : udh::kSmCount * 16), 256, 0, st>>>(I, I_aug, n4);
  int rc = udh::check_launch("normalise_u8");
  if (rc) return rc;
  udh::patches_u8_kernel<<<dim3((P * P + 255) / 256 < 16 ? (P * P + 255) / 256 : 16, B), 256, 0, st>>>(I, I_prime, pts1, I1, I2, patch_origin,
                                                                                                   img_h, img_w, P);
  return udh::check_launch("patches_u8");
}
