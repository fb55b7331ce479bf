// Baseline-JPEG encode on the device, byte-identical to cv2.imencode('.jpg') with libjpeg-turbo's defaults (JFIF, standard
// Huffman tables, ISLOW DCT, YCbCr 4:2:0 for colour, no restart markers).  oracle/jpeg_enc.py restates every stage.
// The quantised DCs are known before any bit is written, so nothing in the entropy coder is serial:
//   enc_coef_kernel   one thread per block of the scan (in MCU order): colour conversion, h2v2 downsampling and edge
//                     replication read straight from the image, ISLOW DCT, reciprocal quantisation; writes the coefficients
//                     (zigzag order) and the bit count of the block's AC codes.  Dummy blocks get zero coefficients here.
//   enc_scan_kernel   one CTA per image: gives every dummy block the DC compress_data gives it, adds each block's DC code
//                     length (the difference to the previous block of its component) and turns the bit counts into bit
//                     offsets with an exclusive scan.
//   enc_write_kernel  one thread per block writes its codes at its bit offset (atomicOr: neighbours share boundary words).
//   enc_stuff_kernel  one CTA per image: header, the stream with 0xFF -> 0xFF 0x00 (a scan over the 0xFF bytes gives each
//                     byte its output position), the final byte padded with 1-bits, EOI, and the file length.
#include <string.h>

#include "common.cuh"

namespace udh {

constexpr int kEncMaxHeader = 624;      // 623 bytes for colour, 328 for gray
constexpr int kEncBlockMaxBits = 11 + 11 + 63 * (16 + 10);   // DC code + bits, 63 AC codes at their longest
constexpr int kEncScanThreads = 1024;

// Everything that depends on (channels, quality) only; passed by value (constant bank).
struct EncParams {
  uint8_t header[kEncMaxHeader];
  int32_t header_len;
  uint16_t recip[2][64], corr[2][64];   // compute_reciprocal of (q << 3), natural order; table 0 luma, 1 chroma
  uint8_t shift[2][64];
  uint16_t dc_code[2][12], ac_code[2][256];
  uint8_t dc_len[2][12], ac_len[2][256];
};

struct EncGeom {
  int32_t h, w, channels;
  int32_t bw, bh;        // luma (or gray) blocks inside the component
  int32_t mw, mh;        // MCUs
  int32_t nblk;          // blocks of the scan, dummies included
  int64_t words;         // 32-bit words of one image's unstuffed stream
  int64_t cap;           // bytes of one output row
};

// Indexed only with unrolled loop counters, so the per-thread coefficient arrays stay in registers
__host__ __device__ constexpr int enc_zigzag(int k) {
  constexpr uint8_t z[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                             41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                             30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
  return z[k];
}

__device__ __forceinline__ int enc_nbits(int v) { return v ? 32 - __clz(v < 0 ? -v : v) : 0; }

// Where block b of the scan lies: component (0 Y, 1 Cb, 2 Cr), block coordinates in that component, whether it is a dummy
struct EncBlock { int comp, bx, by; bool dummy; };
__device__ __forceinline__ EncBlock enc_block(const EncGeom& g, int b) {
  if (g.channels == 1) return {0, b % g.bw, b / g.bw, false};
  const int m = b / 6, k = b - m * 6, my = m / g.mw, mx = m - my * g.mw;
  if (k >= 4) return {k - 3, mx, my, false};
  const int bx = 2 * mx + (k & 1), by = 2 * my + (k >> 1);
  return {0, bx, by, bx >= g.bw || by >= g.bh};
}

// The block of the same component before b in the scan, -1 for the first
__device__ __forceinline__ int enc_prev(const EncGeom& g, int b) {
  if (g.channels == 1) return b - 1;
  const int k = b % 6;
  if (k == 1 || k == 2 || k == 3) return b - 1;
  const int p = b - (k == 0 ? 3 : 6);
  return p >= 0 ? p : -1;
}

// ---- coefficients ------------------------------------------------------------------------------------------------------
// jfdctint.c: CONST_BITS 13, PASS1_BITS 2; rows first (outputs scaled up by PASS1_BITS), columns second
template <bool FIRST>
__device__ __forceinline__ void fdct_1d(int& d0, int& d1, int& d2, int& d3, int& d4, int& d5, int& d6, int& d7) {
  const int t0 = d0 + d7, t7 = d0 - d7, t1 = d1 + d6, t6 = d1 - d6, t2 = d2 + d5, t5 = d2 - d5, t3 = d3 + d4, t4 = d3 - d4;
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  constexpr int S = FIRST ? 11 : 15, R = 1 << (S - 1);
  if (FIRST) {
    d0 = (t10 + t11) * 4;
    d4 = (t10 - t11) * 4;
  } else {
    d0 = (t10 + t11 + 2) >> 2;
    d4 = (t10 - t11 + 2) >> 2;
  }
  int z1 = (t12 + t13) * 4433;
  d2 = (z1 + t13 * 6270 + R) >> S;
  d6 = (z1 - t12 * 15137 + R) >> S;
  z1 = t4 + t7;
  int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const int z5 = (z3 + z4) * 9633;
  const int a4 = t4 * 2446, a5 = t5 * 16819, a6 = t6 * 25172, a7 = t7 * 12299;
  z1 *= -7373; z2 *= -20995; z3 = z3 * -16069 + z5; z4 = z4 * -3196 + z5;
  d7 = (a4 + z1 + z3 + R) >> S;
  d5 = (a5 + z2 + z4 + R) >> S;
  d3 = (a6 + z2 + z3 + R) >> S;
  d1 = (a7 + z1 + z4 + R) >> S;
}

// jccolor.c rgb_ycc_convert of one BGR pixel, component c
__device__ __forceinline__ int enc_ycc(const uint8_t* p, int c) {
  const int b = p[0], g = p[1], r = p[2];
  if (c == 0) return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
  if (c == 1) return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
  return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

__global__ void __launch_bounds__(128) enc_coef_kernel(const uint8_t* __restrict__ img, const EncParams P, const EncGeom g,
                                                       int16_t* __restrict__ coef, uint32_t* __restrict__ bits,
                                                       int32_t* __restrict__ status) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x, n = blockIdx.y;
  if (b >= g.nblk) return;
  int16_t* out = coef + ((int64_t)n * g.nblk + b) * 64;
  const EncBlock e = enc_block(g, b);
  const int t = e.comp ? 1 : 0;
  if (e.dummy) {
#pragma unroll
    for (int k = 0; k < 8; ++k) reinterpret_cast<int4*>(out)[k] = make_int4(0, 0, 0, 0);
    bits[(int64_t)n * g.nblk + b] = P.ac_len[0][0];            // EOB; the DC is set by enc_scan_kernel
    return;
  }
  const uint8_t* src = img + (int64_t)n * g.h * g.w * g.channels;
  int s[64];
  if (g.channels == 1 || e.comp == 0) {                          // full resolution, edges replicated
#pragma unroll
    for (int y = 0; y < 8; ++y) {
      const int yy = min(e.by * 8 + y, g.h - 1);
#pragma unroll
      for (int x = 0; x < 8; ++x) {
        const uint8_t* p = src + ((int64_t)yy * g.w + min(e.bx * 8 + x, g.w - 1)) * g.channels;
        s[y * 8 + x] = (g.channels == 1 ? (int)p[0] : enc_ycc(p, 0)) - 128;
      }
    }
  } else {                                                       // h2v2: the prep controller's rows, the downsampler's columns
    const int last = (g.h + 1) / 2 - 1;
#pragma unroll
    for (int y = 0; y < 8; ++y) {
      const int r = min(e.by * 8 + y, last);
      const uint8_t* r0 = src + (int64_t)(2 * r) * g.w * 3;
      const uint8_t* r1 = src + (int64_t)min(2 * r + 1, g.h - 1) * g.w * 3;
#pragma unroll
      for (int x = 0; x < 8; ++x) {
        const int c0 = min(2 * (e.bx * 8 + x), g.w - 1) * 3, c1 = min(2 * (e.bx * 8 + x) + 1, g.w - 1) * 3;
        const int v = enc_ycc(r0 + c0, e.comp) + enc_ycc(r0 + c1, e.comp) + enc_ycc(r1 + c0, e.comp) + enc_ycc(r1 + c1, e.comp);
        s[y * 8 + x] = ((v + 1 + (x & 1)) >> 2) - 128;
      }
    }
  }
#pragma unroll
  for (int y = 0; y < 8; ++y) fdct_1d<true>(s[y * 8], s[y * 8 + 1], s[y * 8 + 2], s[y * 8 + 3], s[y * 8 + 4], s[y * 8 + 5], s[y * 8 + 6], s[y * 8 + 7]);
#pragma unroll
  for (int x = 0; x < 8; ++x) fdct_1d<false>(s[x], s[8 + x], s[16 + x], s[24 + x], s[32 + x], s[40 + x], s[48 + x], s[56 + x]);
#pragma unroll
  for (int i = 0; i < 64; ++i) {                                 // quantize(): (|x| + corr) * recip >> (16 + shift)
    const uint32_t a = (uint32_t)abs(s[i]);
    const int v = (int)(((a + P.corr[t][i]) * (uint32_t)P.recip[t][i]) >> (16 + P.shift[t][i]));
    s[i] = s[i] < 0 ? -v : v;
  }
  uint32_t nb = 0;
  int run = 0, err = enc_nbits(s[0]) > 11;
#pragma unroll
  for (int k = 1; k < 64; ++k) {
    const int v = s[enc_zigzag(k)];
    if (!v) { ++run; continue; }
    const int sz = enc_nbits(v);
    err |= sz > 10;
    nb += (run >> 4) * P.ac_len[t][0xF0];
    nb += P.ac_len[t][((run & 15) << 4) | min(sz, 10)] + sz;
    run = 0;
  }
  if (run) nb += P.ac_len[t][0];
#pragma unroll
  for (int k = 0; k < 8; ++k) {                                  // int16 pairs, zigzag order
    uint32_t u[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      u[j] = ((uint32_t)s[enc_zigzag(8 * k + 2 * j)] & 0xFFFFu) | ((uint32_t)s[enc_zigzag(8 * k + 2 * j + 1)] << 16);
    reinterpret_cast<int4*>(out)[k] = make_int4((int)u[0], (int)u[1], (int)u[2], (int)u[3]);
  }
  bits[(int64_t)n * g.nblk + b] = nb;
  if (err) atomicCAS(&status[n], 0, 1);                          // not an 8-bit baseline coefficient: cannot happen for uint8 input
}

// ---- bit offsets -------------------------------------------------------------------------------------------------------
// Exclusive scan over the CTA (blockDim.x = kEncScanThreads); `total` = the sum of every thread's v
__device__ __forceinline__ uint32_t enc_block_scan(uint32_t v, uint32_t* sh, uint32_t& total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) sh[wid] = x;
  __syncthreads();
  if (wid == 0) {
    uint32_t w = sh[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    sh[lane] = w;
  }
  __syncthreads();
  const uint32_t pre = wid ? sh[wid - 1] : 0u;
  total = sh[31];
  __syncthreads();                                               // sh is reused by the next call
  return pre + x - v;
}

__device__ __forceinline__ int enc_dc_bits(const EncParams& P, int t, int diff) {
  const int s = enc_nbits(diff);
  return P.dc_len[t][min(s, 11)] + s;
}

__global__ void __launch_bounds__(kEncScanThreads) enc_scan_kernel(const EncParams P, const EncGeom g, int16_t* __restrict__ coef,
                                                                   uint32_t* __restrict__ bits, int64_t* __restrict__ total_bits) {
  __shared__ uint32_t sh[32];
  const int n = blockIdx.x;
  int16_t* c = coef + (int64_t)n * g.nblk * 64;
  uint32_t* off = bits + (int64_t)n * g.nblk;
  if (g.channels == 3 && ((g.bw | g.bh) & 1)) {
    // jccoefct.c compress_data: a dummy block right of the image carries the DC of the block to its left, a dummy row
    // below it the DC of the MCU's last block above; both chains end at a real block of the same MCU
    for (int m = threadIdx.x; m < g.mw * g.mh; m += blockDim.x) {
      int16_t* y = c + (int64_t)m * 6 * 64;
      const int my = m / g.mw, mx = m - my * g.mw;
      const bool right = 2 * mx + 1 >= g.bw, bottom = 2 * my + 1 >= g.bh;
      if (right) y[1 * 64] = y[0];
      if (bottom) y[2 * 64] = y[3 * 64] = y[1 * 64];
      else if (right) y[3 * 64] = y[2 * 64];
    }
    __syncthreads();                                             // the dummies' DCs are visible to the whole CTA
  }
  uint32_t carry = 0;
  for (int b0 = 0; b0 < g.nblk; b0 += blockDim.x) {
    const int b = b0 + threadIdx.x;
    uint32_t v = 0;
    if (b < g.nblk) {
      const int p = enc_prev(g, b);
      const int t = enc_block(g, b).comp ? 1 : 0;
      v = off[b] + enc_dc_bits(P, t, c[(int64_t)b * 64] - (p >= 0 ? c[(int64_t)p * 64] : 0));
    }
    uint32_t tot;
    const uint32_t e = enc_block_scan(v, sh, tot);
    if (b < g.nblk) off[b] = carry + e;
    carry += tot;
  }
  if (threadIdx.x == 0) total_bits[n] = carry;
}

// ---- entropy coding ----------------------------------------------------------------------------------------------------
// Stream words hold the bits MSB first (byte 0 of the stream = bits 31..24 of word 0)
struct EncWriter {
  uint32_t* w;
  uint64_t pos;        // absolute bit position of the next chunk
  uint64_t acc;
  int n;
  __device__ __forceinline__ void chunk(uint32_t v, int len) {   // v left-aligned, len bits valid
    const uint64_t word = pos >> 5;
    const int o = (int)(pos & 31);
    atomicOr(&w[word], v >> o);
    if (o && o + len > 32) atomicOr(&w[word + 1], v << (32 - o));
    pos += len;
  }
  __device__ __forceinline__ void put(uint32_t code, int len) {
    acc = (acc << len) | code;
    n += len;
    if (n >= 32) {
      n -= 32;
      chunk((uint32_t)(acc >> n), 32);
    }
  }
  __device__ __forceinline__ void flush() {
    if (n) chunk((uint32_t)(acc << (32 - n)), n);
  }
};

__global__ void __launch_bounds__(128) enc_write_kernel(const EncParams P, const EncGeom g, const int16_t* __restrict__ coef,
                                                        const uint32_t* __restrict__ bits, const int32_t* __restrict__ status,
                                                        uint32_t* __restrict__ stream) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x, n = blockIdx.y;
  if (b >= g.nblk || status[n]) return;
  const int16_t* c = coef + (int64_t)n * g.nblk * 64;
  const int t = enc_block(g, b).comp ? 1 : 0;
  const int p = enc_prev(g, b);
  int zz[64];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int4 v = __ldg(reinterpret_cast<const int4*>(c + (int64_t)b * 64) + k);
    const int u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      zz[8 * k + 2 * j] = (int)(int16_t)(u[j] & 0xFFFF);
      zz[8 * k + 2 * j + 1] = u[j] >> 16;
    }
  }
  EncWriter wr{stream + (int64_t)n * g.words, bits[(int64_t)n * g.nblk + b], 0, 0};
  const int diff = zz[0] - (p >= 0 ? c[(int64_t)p * 64] : 0);
  int s = enc_nbits(diff);
  wr.put(P.dc_code[t][s], P.dc_len[t][s]);
  if (s) wr.put((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << s) - 1), s);
  int run = 0;
#pragma unroll
  for (int k = 1; k < 64; ++k) {
    const int v = zz[k];
    if (!v) { ++run; continue; }
    for (; run > 15; run -= 16) wr.put(P.ac_code[t][0xF0], P.ac_len[t][0xF0]);
    s = enc_nbits(v);
    const int rs = (run << 4) | s;
    wr.put(P.ac_code[t][rs], P.ac_len[t][rs]);
    wr.put((uint32_t)(v < 0 ? v - 1 : v) & ((1u << s) - 1), s);
    run = 0;
  }
  if (run) wr.put(P.ac_code[t][0], P.ac_len[t][0]);
  wr.flush();
}

// ---- byte stuffing and the file ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kEncScanThreads) enc_stuff_kernel(const EncParams P, const EncGeom g, const uint32_t* __restrict__ stream,
                                                                    const int64_t* __restrict__ total_bits, uint8_t* __restrict__ out,
                                                                    int64_t* __restrict__ nbytes, const int32_t* __restrict__ status) {
  __shared__ uint32_t sh[32];
  const int n = blockIdx.x;
  if (status[n]) {
    if (threadIdx.x == 0) nbytes[n] = 0;
    return;
  }
  uint8_t* o = out + (int64_t)n * g.cap;
  for (int i = threadIdx.x; i < P.header_len; i += blockDim.x) o[i] = P.header[i];
  o += P.header_len;
  const uint32_t* wds = stream + (int64_t)n * g.words;
  const int64_t nbit = total_bits[n], nb = (nbit + 7) >> 3;
  const int padbits = (int)(nbit & 7);
  int64_t carry = 0;                                             // 0xFF bytes before this tile
  for (int64_t j0 = 0; j0 < nb; j0 += 4 * (int64_t)blockDim.x) {
    const int64_t j = j0 + 4 * threadIdx.x;
    uint32_t word = j < nb ? wds[j >> 2] : 0u;
    uint8_t by[4];
    int cnt = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      by[k] = (uint8_t)(word >> (24 - 8 * k));
      if (padbits && j + k == nb - 1) by[k] |= (uint8_t)(0xFFu >> padbits);   // the final byte padded with 1-bits
      cnt += (j + k < nb && by[k] == 0xFF);
    }
    uint32_t tot;
    const uint32_t e = enc_block_scan((uint32_t)cnt, sh, tot);
    int64_t q = j + carry + e;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (j + k >= nb) break;
      o[q++] = by[k];
      if (by[k] == 0xFF) o[q++] = 0;
    }
    carry += tot;
  }
  if (threadIdx.x == 0) {
    o[nb + carry] = 0xFF;
    o[nb + carry + 1] = 0xD9;
    nbytes[n] = P.header_len + nb + carry + 2;
  }
}

// ---- host ------------------------------------------------------------------------------------------------------------------
static const uint8_t kStdLumaQ[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                                      14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                                      18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                                      49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
static const uint8_t kStdChromaQ[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
                                        99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                        99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
static const uint8_t kHostZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                        41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                        30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
// jstdhuff.c: bits[1..16] then the symbols; DC luma, AC luma, DC chroma, AC chroma
static const uint8_t kDcLumaBits[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
static const uint8_t kDcChromaBits[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
static const uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
static const uint8_t kAcLumaBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d};
static const uint8_t kAcLumaVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
    0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
    0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
    0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
    0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
    0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
static const uint8_t kAcChromaBits[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77};
static const uint8_t kAcChromaVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
    0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
    0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
    0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
    0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
    0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
    0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
    0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

// jchuff.c jpeg_make_c_derived_tbl: canonical codes in symbol order
static void enc_codes(const uint8_t* bits, const uint8_t* vals, uint16_t* code, uint8_t* len) {
  int c = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    for (int i = 0; i < bits[l - 1]; ++i, ++k, ++c) {
      code[vals[k]] = (uint16_t)c;
      len[vals[k]] = (uint8_t)l;
    }
    c <<= 1;
  }
}

// jcdctmgr.c compute_reciprocal with a 16-bit DCTELEM
static void enc_reciprocal(int divisor, uint16_t& recip, uint16_t& corr, uint8_t& shift) {
  int b = 31 - __builtin_clz((unsigned)divisor);
  int r = 16 + b;
  uint32_t fq = (1u << r) / (uint32_t)divisor, fr = (1u << r) % (uint32_t)divisor;
  uint32_t c = (uint32_t)divisor / 2;
  if (fr == 0) {
    fq >>= 1;
    --r;
  } else if (fr <= (uint32_t)divisor / 2) {
    ++c;
  } else {
    ++fq;
  }
  recip = (uint16_t)fq;
  corr = (uint16_t)c;
  shift = (uint8_t)(r - 16);
}

static int enc_header(int h, int w, int channels, const uint8_t (*qt)[64], uint8_t* o) {
  int p = 0;
  auto seg = [&](int marker, int len) { o[p++] = 0xFF; o[p++] = (uint8_t)marker; o[p++] = (uint8_t)((len + 2) >> 8); o[p++] = (uint8_t)((len + 2) & 255); };
  o[p++] = 0xFF; o[p++] = 0xD8;
  static const uint8_t jfif[14] = {'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
  seg(0xE0, 14);
  memcpy(o + p, jfif, 14); p += 14;
  const int nt = channels == 3 ? 2 : 1;
  for (int t = 0; t < nt; ++t) {
    seg(0xDB, 65);
    o[p++] = (uint8_t)t;
    for (int k = 0; k < 64; ++k) o[p++] = qt[t][kHostZigzag[k]];
  }
  seg(0xC0, 6 + 3 * channels);
  o[p++] = 8; o[p++] = (uint8_t)(h >> 8); o[p++] = (uint8_t)h; o[p++] = (uint8_t)(w >> 8); o[p++] = (uint8_t)w; o[p++] = (uint8_t)channels;
  for (int c = 0; c < channels; ++c) {
    o[p++] = (uint8_t)(c + 1);
    o[p++] = channels == 3 && c == 0 ? 0x22 : 0x11;
    o[p++] = c ? 1 : 0;
  }
  const uint8_t* bits[2][2] = {{kDcLumaBits, kAcLumaBits}, {kDcChromaBits, kAcChromaBits}};
  const uint8_t* vals[2][2] = {{kDcVals, kAcLumaVals}, {kDcVals, kAcChromaVals}};
  for (int t = 0; t < nt; ++t)
    for (int cls = 0; cls < 2; ++cls) {
      int nv = 0;
      for (int l = 0; l < 16; ++l) nv += bits[t][cls][l];
      seg(0xC4, 17 + nv);
      o[p++] = (uint8_t)(cls << 4 | t);
      memcpy(o + p, bits[t][cls], 16); p += 16;
      memcpy(o + p, vals[t][cls], nv); p += nv;
    }
  seg(0xDA, 4 + 2 * channels);
  o[p++] = (uint8_t)channels;
  for (int c = 0; c < channels; ++c) { o[p++] = (uint8_t)(c + 1); o[p++] = c ? 0x11 : 0x00; }
  o[p++] = 0; o[p++] = 63; o[p++] = 0;
  return p;
}

static void enc_params(int h, int w, int channels, int quality, EncParams& P) {
  memset(&P, 0, sizeof(P));
  const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;   // jpeg_quality_scaling
  uint8_t qt[2][64];
  for (int i = 0; i < 64; ++i) {                                          // jpeg_add_quant_table, force_baseline
    const int base[2] = {kStdLumaQ[i], kStdChromaQ[i]};
    for (int t = 0; t < 2; ++t) {
      int v = (base[t] * scale + 50) / 100;
      qt[t][i] = (uint8_t)(v < 1 ? 1 : v > 255 ? 255 : v);
      enc_reciprocal(qt[t][i] << 3, P.recip[t][i], P.corr[t][i], P.shift[t][i]);
    }
  }
  P.header_len = enc_header(h, w, channels, qt, P.header);
  enc_codes(kDcLumaBits, kDcVals, P.dc_code[0], P.dc_len[0]);
  enc_codes(kDcChromaBits, kDcVals, P.dc_code[1], P.dc_len[1]);
  enc_codes(kAcLumaBits, kAcLumaVals, P.ac_code[0], P.ac_len[0]);
  enc_codes(kAcChromaBits, kAcChromaVals, P.ac_code[1], P.ac_len[1]);
}

static bool enc_geom(int h, int w, int channels, EncGeom& g) {
  if (h < 1 || w < 1 || h > 65535 || w > 65535 || (channels != 1 && channels != 3)) return false;
  g.h = h; g.w = w; g.channels = channels;
  g.bw = (w + 7) / 8; g.bh = (h + 7) / 8;
  if (channels == 3) {
    g.mw = (w + 15) / 16; g.mh = (h + 15) / 16;
    g.nblk = 6 * g.mw * g.mh;
  } else {
    g.mw = g.bw; g.mh = g.bh;
    g.nblk = g.bw * g.bh;
  }
  const int64_t maxbits = (int64_t)g.nblk * kEncBlockMaxBits;
  if (maxbits >= ((int64_t)1 << 32)) return false;                 // bit offsets are 32-bit
  g.words = (maxbits + 31) / 32 + 1;
  uint8_t hdr[kEncMaxHeader], q[2][64] = {};
  g.cap = enc_header(h, w, channels, q, hdr) + 2 * ((maxbits + 7) / 8) + 2;   // header, stream with every byte stuffed, EOI
  return true;
}

static size_t enc_align(size_t x) { return (x + 255) / 256 * 256; }

}  // namespace udh

using namespace udh;

extern "C" int64_t udh_jpeg_encode_capacity(int h, int w, int channels) {
  EncGeom g;
  return enc_geom(h, w, channels, g) ? g.cap : 0;
}

extern "C" size_t udh_jpeg_encode_workspace_bytes(int n, int h, int w, int channels) {
  EncGeom g;
  if (n < 1 || !enc_geom(h, w, channels, g)) return 0;
  return enc_align((size_t)n * g.nblk * 64 * sizeof(int16_t)) + enc_align((size_t)n * g.nblk * sizeof(uint32_t)) +
         enc_align((size_t)n * sizeof(int64_t)) + (size_t)n * g.words * sizeof(uint32_t);
}

extern "C" int udh_jpeg_encode(const uint8_t* img, int n, int h, int w, int channels, int quality, uint8_t* out, int64_t cap,
                               int64_t* nbytes, int32_t* status, void* ws, size_t ws_bytes, void* stream) {
  UDH_REQUIRE(img && out && nbytes && status && ws, "udh_jpeg_encode: null pointer");
  EncGeom g;
  UDH_REQUIRE(n >= 1 && n <= 65535 && enc_geom(h, w, channels, g), "udh_jpeg_encode: bad dimensions (n %d, %dx%d, %d channels)", n, h, w, channels);
  UDH_REQUIRE(quality >= 1 && quality <= 100, "udh_jpeg_encode: quality %d outside 1..100", quality);
  UDH_REQUIRE(cap >= g.cap, "udh_jpeg_encode: cap %lld below the capacity %lld", (long long)cap, (long long)g.cap);
  const size_t need = udh_jpeg_encode_workspace_bytes(n, h, w, channels);
  if (ws_bytes < need) {
    set_error("udh_jpeg_encode: workspace of %zu bytes, %zu needed", ws_bytes, need);
    return UDH_EWS;
  }
  UDH_REQUIRE(((uintptr_t)ws & 15) == 0, "udh_jpeg_encode: workspace must be 16-byte aligned");
  g.cap = cap;
  EncParams P;
  enc_params(h, w, channels, quality, P);
  cudaStream_t st = as_stream(stream);
  uint8_t* p = static_cast<uint8_t*>(ws);
  int16_t* coef = reinterpret_cast<int16_t*>(p);
  p += enc_align((size_t)n * g.nblk * 64 * sizeof(int16_t));
  uint32_t* bits = reinterpret_cast<uint32_t*>(p);
  p += enc_align((size_t)n * g.nblk * sizeof(uint32_t));
  int64_t* total = reinterpret_cast<int64_t*>(p);
  p += enc_align((size_t)n * sizeof(int64_t));
  uint32_t* stream_words = reinterpret_cast<uint32_t*>(p);
  UDH_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t) * n, st));
  UDH_CUDA(cudaMemsetAsync(stream_words, 0, (size_t)n * g.words * sizeof(uint32_t), st));
  const dim3 grid((g.nblk + 127) / 128, n);
  enc_coef_kernel<<<grid, 128, 0, st>>>(img, P, g, coef, bits, status);
  int rc = check_launch("enc_coef");
  if (rc) return rc;
  enc_scan_kernel<<<n, kEncScanThreads, 0, st>>>(P, g, coef, bits, total);
  if ((rc = check_launch("enc_scan"))) return rc;
  enc_write_kernel<<<grid, 128, 0, st>>>(P, g, coef, bits, status, stream_words);
  if ((rc = check_launch("enc_write"))) return rc;
  enc_stuff_kernel<<<n, kEncScanThreads, 0, st>>>(P, g, stream_words, total, out, nbytes, status);
  return check_launch("udh_jpeg_encode");
}
