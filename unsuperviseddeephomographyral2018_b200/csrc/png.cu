// PNG decode on the device, bit-identical to cv2.imread(..., IMREAD_COLOR) for the files the host parser accepts
// (non-interlaced, 8-bit gray / RGB / RGBA, no chunk that changes what cv2 returns; see include/udh.h).
//   host parser          checks the signature, IHDR and every chunk's CRC, and lists the IDAT payloads; udh_png_plan
//                        concatenates each file's payloads, so its zlib stream is contiguous in the IDAT buffer.
//   png_inflate_kernel   one CTA per zlib stream.  Thread 0 decodes the Huffman codes serially: literals go straight to
//                        the filtered-scanline buffer, matches and stored blocks become tokens in shared memory.  When
//                        the token buffer is full (or the stream ends) the CTA expands the tokens in parallel, batch by
//                        batch: a batch is a run of tokens none of whose sources overlaps another token of the batch, so
//                        its tokens are copied at once (one warp per token, or the whole CTA for a batch of one).  A
//                        match that overlaps its own output (distance < length) copies byte j from position
//                        src + j mod distance, which is written before the match starts.  Then the CTA checks the
//                        Adler-32 of the output.
//   png_unfilter_kernel  one CTA per image, rows in order through two shared-memory rows: None and Up are parallel
//                        across bytes, Sub / Average / Paeth run one thread per channel along the row.  The store
//                        replicates gray to three channels, drops alpha and writes BGR (or RGB).
// Any malformed stream ends its image with a UDH_PNG_E_* status; no access leaves the image's input or output.
#include <stddef.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace udh {

struct PngImage {
  int64_t src, len;   // zlib stream: [src, src + len) of the IDAT buffer
  int64_t raw;        // filtered scanlines: [raw, raw + h * (1 + w * ch)) of the workspace
  int32_t ch, pad;    // samples per pixel (1, 3 or 4)
};

struct PngPlanHeader {
  uint32_t magic;
  int32_t n, h, w;
  int64_t raw_bytes, idat_bytes;
  int32_t max_row, pad[3];   // the longest row's samples (w * ch)
};

static_assert(sizeof(PngImage) % 16 == 0 && sizeof(PngPlanHeader) % 16 == 0, "plan sections must stay 16-byte aligned");

constexpr uint32_t kPngMagic = 0x504e4731u;
constexpr int kPngThreads = 128;
constexpr int kPngTokens = 1024;   // tokens per expansion round
constexpr int kPngLutBits = 9;

// ---- device: inflate ----------------------------------------------------------------------------------------------------
// canonical Huffman code: a 9-bit lookup ((length << 9) | symbol, 0 = longer code or none) and puff's count / symbol lists
struct PngHuff {
  uint16_t lut[1 << kPngLutBits];
  int16_t count[16];
  int16_t sym[288];
};

struct PngToken {
  int32_t dst;   // output position
  int32_t len;   // > 0: a match from output position src; < 0: a stored block of -len bytes from input offset src
  int32_t src;
};

// LSB-first bit reader over one zlib stream; bytes past the end read as zero, and bad() tells when they were consumed
struct InflateBits {
  const uint8_t* base;
  int64_t len, next;
  uint64_t acc;
  int n;

  __device__ __forceinline__ void fill() {
    while (n <= 56) {
      const uint64_t b = next < len ? (uint64_t)__ldg(base + next) : 0;
      ++next;
      acc |= b << n;
      n += 8;
    }
  }
  __device__ __forceinline__ uint32_t bits(int k) {   // k <= 32, k <= n
    const uint32_t v = (uint32_t)(acc & ((1ull << k) - 1));
    acc >>= k;
    n -= k;
    return v;
  }
  __device__ __forceinline__ void drop(int k) { acc >>= k; n -= k; }
  __device__ __forceinline__ int64_t consumed() const { return next * 8 - n; }
  __device__ __forceinline__ bool bad() const { return consumed() > len * 8; }
};

__device__ __forceinline__ int png_decode_sym(InflateBits& br, const PngHuff& h) {
  const uint32_t e = h.lut[br.acc & ((1u << kPngLutBits) - 1)];
  if (e) {
    br.drop(e >> kPngLutBits);
    return e & ((1u << kPngLutBits) - 1);
  }
  int code = 0, first = 0, index = 0;
  for (int l = 1; l <= 15; ++l) {
    code |= (int)((br.acc >> (l - 1)) & 1);
    const int count = h.count[l];
    if (code - count < first) {
      br.drop(l);
      return h.sym[index + (code - first)];
    }
    index += count;
    first = (first + count) << 1;
    code <<= 1;
  }
  return -1;
}

// zlib's inflate_table rules: over-subscribed codes are invalid; incomplete ones too, except a single code of length 1
// in the literal/length and distance codes; a code without symbols is valid (every decode with it fails).
__device__ bool png_build(PngHuff& h, const uint8_t* lens, int n, bool codes, int16_t* offs) {
  for (int l = 0; l < 16; ++l) h.count[l] = 0;
  for (int s = 0; s < n; ++s) ++h.count[lens[s]];
  uint32_t* lut = reinterpret_cast<uint32_t*>(h.lut);
  for (int j = 0; j < (1 << kPngLutBits) / 2; ++j) lut[j] = 0;
  int max = 15;
  while (max >= 1 && h.count[max] == 0) --max;
  h.count[0] = 0;
  if (max == 0) return true;
  int left = 1;
  for (int l = 1; l <= 15; ++l) {
    left = (left << 1) - h.count[l];
    if (left < 0) return false;
  }
  if (left > 0 && (codes || max != 1)) return false;
  offs[1] = 0;
  for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + h.count[l];
  for (int s = 0; s < n; ++s)
    if (lens[s]) h.sym[offs[lens[s]]++] = (int16_t)s;
  int code = 0, idx = 0;
  for (int l = 1; l <= 15; ++l) {
    for (int i = 0; i < h.count[l]; ++i, ++code, ++idx) {
      if (l > kPngLutBits) continue;
      const uint16_t e = (uint16_t)((l << kPngLutBits) | h.sym[idx]);
      for (uint32_t j = __brev((uint32_t)code) >> (32 - l); j < (1u << kPngLutBits); j += 1u << l) h.lut[j] = e;
    }
    code <<= 1;
  }
  return true;
}

__constant__ uint16_t c_len_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
                                        131, 163, 195, 227, 258};
__constant__ uint8_t c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dist_base[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537,
                                         2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_cl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

struct InflateShared {
  PngHuff lit, dist;
  uint8_t lens[320];
  int16_t offs[16];
  PngToken tok[kPngTokens];
  uint16_t bstart[kPngTokens + 1];
  int32_t ntok, nbatch, state;   // state: 0 running, 1 stream complete, < 0 -UDH_PNG_E_*
  uint32_t adler;
  unsigned long long sa[kPngThreads / 32], sb[kPngThreads / 32];
};

// thread 0's decoder: everything that survives from one expansion round to the next
struct InflateState {
  InflateBits br;
  int64_t op;           // bytes output so far
  int32_t wsize;        // the window the zlib header declares
  int32_t inblock, final;
  int32_t bfirst, bend; // current batch: first token's output position, end of its last token's output
};

__device__ __forceinline__ int png_dynamic(InflateState& S, InflateShared& sm) {
  InflateBits& br = S.br;
  br.fill();
  const int nlen = br.bits(5) + 257, ndist = br.bits(5) + 1, ncode = br.bits(4) + 4;
  if (nlen > 286 || ndist > 30) return UDH_PNG_E_BLOCK;
  for (int i = 0; i < 19; ++i) sm.lens[i] = 0;
  for (int i = 0; i < ncode; ++i) {
    br.fill();
    sm.lens[c_cl_order[i]] = (uint8_t)br.bits(3);
  }
  if (br.bad()) return UDH_PNG_E_TRUNCATED;
  if (!png_build(sm.lit, sm.lens, 19, true, sm.offs)) return UDH_PNG_E_BLOCK;
  int index = 0;
  while (index < nlen + ndist) {
    br.fill();
    const int sym = png_decode_sym(br, sm.lit);
    if (sym < 0) return br.bad() ? UDH_PNG_E_TRUNCATED : UDH_PNG_E_BLOCK;
    if (sym < 16) {
      sm.lens[index++] = (uint8_t)sym;
    } else {
      int len = 0, rep;
      if (sym == 16) {
        if (index == 0) return UDH_PNG_E_BLOCK;
        len = sm.lens[index - 1];
        rep = 3 + br.bits(2);
      } else if (sym == 17) {
        rep = 3 + br.bits(3);
      } else {
        rep = 11 + br.bits(7);
      }
      if (index + rep > nlen + ndist) return UDH_PNG_E_BLOCK;
      while (rep--) sm.lens[index++] = (uint8_t)len;
    }
    if (br.bad()) return UDH_PNG_E_TRUNCATED;
  }
  if (sm.lens[256] == 0) return UDH_PNG_E_BLOCK;   // no end-of-block code
  if (!png_build(sm.lit, sm.lens, nlen, false, sm.offs)) return UDH_PNG_E_BLOCK;
  if (!png_build(sm.dist, sm.lens + nlen, ndist, false, sm.offs)) return UDH_PNG_E_BLOCK;
  return 0;
}

__device__ __forceinline__ void png_fixed(InflateShared& sm) {
  for (int i = 0; i < 288; ++i) sm.lens[i] = i < 144 ? 8 : (i < 256 ? 9 : (i < 280 ? 7 : 8));
  png_build(sm.lit, sm.lens, 288, false, sm.offs);
  for (int i = 0; i < 32; ++i) sm.lens[i] = 5;
  png_build(sm.dist, sm.lens, 32, false, sm.offs);
}

__device__ __forceinline__ void png_emit(InflateState& S, InflateShared& sm, int dst, int len, int src, int src_lo, int src_hi) {
  // a new batch unless the source lies wholly before the batch's first output or wholly after its last one
  const int t = sm.ntok;
  if (t == 0 || !(src_hi <= S.bfirst || src_lo >= S.bend)) {
    sm.bstart[sm.nbatch++] = (uint16_t)t;
    S.bfirst = dst;
  }
  sm.tok[t] = PngToken{dst, len, src};
  sm.ntok = t + 1;
  S.bend = dst + (len < 0 ? -len : len);
}

// Decode until the token buffer is full, the stream ends or an error; returns the new state (0, 1 or -UDH_PNG_E_*).
__device__ __forceinline__ int png_decode_round(InflateState& S, InflateShared& sm, uint8_t* out, int64_t outlen) {
  InflateBits& br = S.br;
  sm.ntok = 0;
  sm.nbatch = 0;
  while (sm.ntok < kPngTokens) {
    if (!S.inblock) {
      if (S.final) {   // the Adler-32, big-endian, at the next byte boundary
        br.fill();
        br.drop(br.n & 7);
        uint32_t a = 0;
        for (int i = 0; i < 4; ++i) a = (a << 8) | br.bits(8);
        if (br.bad()) return -UDH_PNG_E_TRUNCATED;
        if (S.op != outlen) return -UDH_PNG_E_SHORT;
        sm.adler = a;
        return 1;
      }
      br.fill();
      S.final = br.bits(1);
      const int type = br.bits(2);
      if (type == 0) {
        br.drop(br.n & 7);
        const uint32_t len = br.bits(16), nlen = br.bits(16);
        if (br.bad()) return -UDH_PNG_E_TRUNCATED;
        if (len != (~nlen & 0xffffu)) return -UDH_PNG_E_BLOCK;
        const int64_t pos = br.consumed() >> 3;
        if (pos + len > br.len) return -UDH_PNG_E_TRUNCATED;
        if (S.op + len > outlen) return -UDH_PNG_E_LONG;
        if (len) png_emit(S, sm, (int)S.op, -(int)len, (int)pos, 0, 0);
        S.op += len;
        br.next = pos + len;   // restart the reader after the stored bytes
        br.acc = 0;
        br.n = 0;
      } else if (type == 1) {
        png_fixed(sm);
        S.inblock = 1;
      } else if (type == 2) {
        const int e = png_dynamic(S, sm);
        if (e) return -e;
        S.inblock = 1;
      } else {
        return -UDH_PNG_E_BLOCK;
      }
      continue;
    }
    br.fill();
    int sym = png_decode_sym(br, sm.lit);
    if (sym < 0) return br.bad() ? -UDH_PNG_E_TRUNCATED : -UDH_PNG_E_CODE;
    if (sym < 256) {
      if (br.bad()) return -UDH_PNG_E_TRUNCATED;
      if (S.op >= outlen) return -UDH_PNG_E_LONG;
      out[S.op++] = (uint8_t)sym;
    } else if (sym == 256) {
      if (br.bad()) return -UDH_PNG_E_TRUNCATED;
      S.inblock = 0;
    } else {
      sym -= 257;
      if (sym >= 29) return -UDH_PNG_E_CODE;
      const int len = c_len_base[sym] + (int)br.bits(c_len_extra[sym]);
      const int ds = png_decode_sym(br, sm.dist);
      if (ds < 0 || ds >= 30) return br.bad() ? -UDH_PNG_E_TRUNCATED : -UDH_PNG_E_CODE;
      const int dist = c_dist_base[ds] + (int)br.bits(c_dist_extra[ds]);
      if (br.bad()) return -UDH_PNG_E_TRUNCATED;
      if (dist > S.op || dist > S.wsize) return -UDH_PNG_E_DISTANCE;
      if (S.op + len > outlen) return -UDH_PNG_E_LONG;
      const int dst = (int)S.op, src = dst - dist;
      png_emit(S, sm, dst, len, src, src, src + min(dist, len));
      S.op += len;
    }
  }
  return 0;
}

__global__ void __launch_bounds__(kPngThreads) png_inflate_kernel(const PngImage* __restrict__ imgs, const uint8_t* __restrict__ idat,
                                                                  uint8_t* raw, int32_t* status, int h, int w) {
  __shared__ InflateShared sm;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const PngImage im = imgs[blockIdx.x];
  const int64_t outlen = (int64_t)h * (1 + (int64_t)w * im.ch);
  uint8_t* out = raw + im.raw;
  const uint8_t* in = idat + im.src;
  InflateState S;
  if (tid == 0) {
    S.br.base = in;
    S.br.len = im.len;
    S.br.next = 0;
    S.br.acc = 0;
    S.br.n = 0;
    S.op = 0;
    S.inblock = S.final = 0;
    S.bfirst = S.bend = 0;
    S.br.fill();
    const uint32_t cmf = S.br.bits(8), flg = S.br.bits(8);
    S.wsize = 1 << ((cmf >> 4) + 8);
    if (S.br.bad()) sm.state = -UDH_PNG_E_TRUNCATED;
    else if ((cmf & 15) != 8 || (cmf >> 4) > 7 || ((cmf << 8) | flg) % 31 != 0 || (flg & 0x20)) sm.state = -UDH_PNG_E_ZLIB;
    else sm.state = 0;
    sm.ntok = sm.nbatch = 0;
  }
  __syncthreads();
  while (sm.state == 0) {
    __syncthreads();   // every thread has read the state before thread 0 starts the next round
    if (tid == 0) {
      sm.state = png_decode_round(S, sm, out, outlen);
      sm.bstart[sm.nbatch] = (uint16_t)sm.ntok;
    }
    __syncthreads();
    for (int b = 0; b < sm.nbatch; ++b) {
      const int t0 = sm.bstart[b], t1 = sm.bstart[b + 1];
      const bool whole = t1 - t0 == 1;   // a batch of one token: the whole CTA copies it
      for (int t = t0 + (whole ? 0 : warp); t < t1; t += kPngThreads / 32) {
        const PngToken T = sm.tok[t];
        const int r = whole ? tid : lane, step = whole ? kPngThreads : 32;
        if (T.len < 0) {
          for (int j = r; j < -T.len; j += step) out[T.dst + j] = __ldg(in + T.src + j);
        } else {
          const int d = T.dst - T.src;
          if (d >= T.len)
            for (int j = r; j < T.len; j += step) out[T.dst + j] = out[T.src + j];
          else
            for (int j = r; j < T.len; j += step) out[T.dst + j] = out[T.src + j % d];
        }
        if (whole) break;
      }
      __syncthreads();
    }
  }
  if (sm.state < 0) {
    if (tid == 0) status[blockIdx.x] = -sm.state;
    return;
  }
  // Adler-32: A = 1 + sum d_i, B = n + sum (n - i) d_i (mod 65521)
  unsigned long long a = 0, b = 0;
  for (int64_t i = tid; i < outlen; i += kPngThreads) {
    const uint32_t d = out[i];
    a += d;
    b += (unsigned long long)((outlen - i) % 65521) * d;
  }
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  if (lane == 0) {
    sm.sa[warp] = a;
    sm.sb[warp] = b;
  }
  __syncthreads();
  if (tid == 0) {
    unsigned long long A = 1, B = (unsigned long long)(outlen % 65521);
    for (int k = 0; k < kPngThreads / 32; ++k) {
      A += sm.sa[k];
      B += sm.sb[k];
    }
    const uint32_t adler = (uint32_t)((B % 65521) << 16 | (A % 65521));
    if (adler != sm.adler) status[blockIdx.x] = UDH_PNG_E_ADLER;
  }
}

// ---- device: unfilter + convert -----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kPngThreads) png_unfilter_kernel(const PngImage* __restrict__ imgs, const uint8_t* __restrict__ raw,
                                                                   int32_t* status, uint8_t* __restrict__ out, int h, int w, int rowcap,
                                                                   int rgb) {
  extern __shared__ uint8_t rows[];
  const int k = blockIdx.x, tid = threadIdx.x;
  if (status[k]) return;
  const PngImage im = imgs[k];
  const int ch = im.ch, rb = w * ch;
  uint8_t* prev = rows;
  uint8_t* cur = rows + rowcap;
  for (int i = tid; i < rb; i += kPngThreads) prev[i] = 0;
  uint8_t* dst = out + (int64_t)k * h * w * 3;
  const int r0 = rgb ? 0 : 2, r2 = rgb ? 2 : 0;
  for (int y = 0; y < h; ++y) {
    const uint8_t* src = raw + im.raw + (int64_t)y * (rb + 1);
    const int f = src[0];
    if (f > 4) {
      if (tid == 0) status[k] = UDH_PNG_E_FILTER;
      return;
    }
    for (int i = tid; i < rb; i += kPngThreads) {
      int v = src[1 + i];
      if (f == 2) v += prev[i];
      cur[i] = (uint8_t)v;
    }
    __syncthreads();
    if (f != 0 && f != 2 && tid < ch) {
      int a = 0, c = 0;   // the reconstructed byte to the left and the one above it
      for (int i = tid; i < rb; i += ch) {
        const int x = cur[i], b = prev[i];
        int pred;
        if (f == 1) {
          pred = a;
        } else if (f == 3) {
          pred = (a + b) >> 1;
        } else {
          const int pa = abs(b - c), pb = abs(a - c), pc = abs(a + b - 2 * c);
          pred = (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
        }
        a = (x + pred) & 255;
        c = b;
        cur[i] = (uint8_t)a;
      }
    }
    __syncthreads();
    uint8_t* drow = dst + (int64_t)y * w * 3;
    for (int x = tid; x < w; x += kPngThreads) {
      const uint8_t* p = cur + x * ch;
      const uint8_t v0 = p[0], v1 = ch >= 3 ? p[1] : v0, v2 = ch >= 3 ? p[2] : v0;
      drow[3 * x + r0] = v0;
      drow[3 * x + 1] = v1;
      drow[3 * x + r2] = v2;
    }
    uint8_t* t = prev;
    prev = cur;
    cur = t;
  }
}

// ---- host: parser and plan ----------------------------------------------------------------------------------------------
// CRC-32 (ISO-HDLC, the PNG chunk CRC), slicing by 8: the parser checks every byte of every file once
static uint32_t g_crc_table[8][256];
static struct CrcInit {
  CrcInit() {
    for (uint32_t n = 0; n < 256; ++n) {
      uint32_t c = n;
      for (int k = 0; k < 8; ++k) c = (c & 1) ? 0xedb88320u ^ (c >> 1) : c >> 1;
      g_crc_table[0][n] = c;
    }
    for (uint32_t n = 0; n < 256; ++n)
      for (int k = 1; k < 8; ++k) g_crc_table[k][n] = g_crc_table[0][g_crc_table[k - 1][n] & 255] ^ (g_crc_table[k - 1][n] >> 8);
  }
} g_crc_init;

static uint32_t png_crc(const uint8_t* p, int64_t n) {
  uint32_t c = 0xffffffffu;
  const uint32_t(*t)[256] = g_crc_table;
  for (; n >= 8; n -= 8, p += 8) {
    uint32_t a, b;
    memcpy(&a, p, 4);
    memcpy(&b, p + 4, 4);
    a ^= c;   // little-endian host
    c = t[7][a & 255] ^ t[6][(a >> 8) & 255] ^ t[5][(a >> 16) & 255] ^ t[4][a >> 24] ^ t[3][b & 255] ^ t[2][(b >> 8) & 255] ^
        t[1][(b >> 16) & 255] ^ t[0][b >> 24];
  }
  for (; n > 0; --n) c = t[0][(c ^ *p++) & 255] ^ (c >> 8);
  return c ^ 0xffffffffu;
}

static inline int64_t align_up_png(int64_t x) { return (x + 15) / 16 * 16; }

static inline uint32_t be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }

struct PngParsed {
  udh_png_info info;
  std::vector<std::pair<int64_t, int64_t>> idat;   // (offset in the file, length) of each IDAT payload
};

static bool png_type_is(const uint8_t* t, const char* s) { return memcmp(t, s, 4) == 0; }

// ancillary chunks cv2.imread(IMREAD_COLOR) does not act on
static bool png_ignored_chunk(const uint8_t* t) {
  return png_type_is(t, "tEXt") || png_type_is(t, "zTXt") || png_type_is(t, "iTXt") || png_type_is(t, "tIME") || png_type_is(t, "pHYs");
}

static int png_parse_impl(const uint8_t* d, int64_t n, PngParsed& P, bool check_crc = true) {
  static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
  memset(&P.info, 0, sizeof(P.info));
  P.idat.clear();
  if (n >= 3 && d[0] == 0xff && d[1] == 0xd8 && d[2] == 0xff) return UDH_PNG_R_JPEG;
  if (n < 8 || memcmp(d, sig, 8) != 0) return UDH_PNG_R_NOT_PNG;
  int64_t pos = 8;
  bool ihdr = false, iend = false, idat_closed = false, other = false;
  while (pos < n) {
    if (n - pos < 8) return UDH_PNG_R_TRUNCATED;
    const uint32_t len = be32(d + pos);
    const uint8_t* type = d + pos + 4;
    if (len > 0x7fffffffu) return UDH_PNG_R_MALFORMED;
    if ((int64_t)len + 12 > n - pos) return png_type_is(type, "IDAT") ? UDH_PNG_R_IDAT_TRUNCATED : UDH_PNG_R_TRUNCATED;
    if (check_crc && png_crc(type, (int64_t)len + 4) != be32(d + pos + 8 + len)) return UDH_PNG_R_CRC;
    const uint8_t* body = d + pos + 8;
    if (!ihdr) {
      if (!png_type_is(type, "IHDR") || len != 13) return UDH_PNG_R_MALFORMED;
      udh_png_info& I = P.info;
      const uint32_t wd = be32(body), ht = be32(body + 4);
      I.bit_depth = body[8];
      I.color_type = body[9];
      I.interlace = body[12];
      if (wd == 0 || ht == 0 || wd > 0x7fffffffu || ht > 0x7fffffffu || body[10] != 0 || body[11] != 0 || I.interlace > 1)
        return UDH_PNG_R_MALFORMED;
      I.width = (int32_t)wd;
      I.height = (int32_t)ht;
      const int dp = I.bit_depth, ct = I.color_type;
      const bool ok = (ct == 0 && (dp == 1 || dp == 2 || dp == 4 || dp == 8 || dp == 16)) ||
                      (ct == 3 && (dp == 1 || dp == 2 || dp == 4 || dp == 8)) ||
                      ((ct == 2 || ct == 4 || ct == 6) && (dp == 8 || dp == 16));
      if (!ok) return UDH_PNG_R_MALFORMED;
      I.channels = ct == 2 ? 3 : (ct == 4 ? 2 : (ct == 6 ? 4 : 1));
      ihdr = true;
    } else if (png_type_is(type, "IDAT")) {
      if (idat_closed) return UDH_PNG_R_MALFORMED;   // IDAT chunks must be consecutive
      P.idat.emplace_back(pos + 8, (int64_t)len);
      P.info.idat_bytes += len;
    } else if (png_type_is(type, "IEND")) {
      iend = true;
      break;
    } else if (png_type_is(type, "IHDR")) {
      return UDH_PNG_R_MALFORMED;
    } else if (!png_ignored_chunk(type)) {
      other = true;
    }
    if (!P.idat.empty() && !png_type_is(type, "IDAT")) idat_closed = true;
    pos += (int64_t)len + 12;
  }
  if (!iend) return UDH_PNG_R_NO_IEND;
  if (!ihdr || P.idat.empty()) return UDH_PNG_R_MALFORMED;
  const udh_png_info& I = P.info;
  if (I.color_type == 3) return UDH_PNG_R_PALETTE;
  if (I.bit_depth == 16) return UDH_PNG_R_DEPTH16;
  if (I.bit_depth < 8) return UDH_PNG_R_DEPTH_SUB8;
  if (I.interlace) return UDH_PNG_R_INTERLACED;
  if (I.color_type == 4) return UDH_PNG_R_GRAY_ALPHA;
  if (other) return UDH_PNG_R_CHUNK;
  return UDH_PNG_R_OK;
}

// parsed == nullptr: sizing only (udh_png_plan_bytes), without the CRCs; udh_png_plan checks every file in full before it
// writes anything
static int png_build_plan(const uint8_t* data, const int64_t* offsets, int n, int h, int w, std::vector<PngImage>& imgs,
                          std::vector<PngParsed>* parsed, int64_t* raw_bytes, int64_t* idat_bytes, int* max_row) {
  imgs.resize(n);
  if (parsed) parsed->resize(n);
  PngParsed P;
  int64_t raw = 0, src = 0;
  *max_row = 0;
  for (int k = 0; k < n; ++k) {
    const int64_t b = offsets[k], len = offsets[k + 1] - offsets[k];
    if (len < 0) {
      set_error("udh_png_plan: offsets must not decrease (image %d)", k);
      return UDH_EINVAL;
    }
    const int r = png_parse_impl(data + b, len, P, parsed != nullptr);
    if (r != UDH_PNG_R_OK) {
      set_error("udh_png_plan: image %d is not supported (reason %d)", k, r);
      return UDH_ENOSUP;
    }
    if (P.info.height != h || P.info.width != w) {
      set_error("udh_png_plan: image %d is %dx%d, the plan is for %dx%d", k, P.info.height, P.info.width, h, w);
      return UDH_EINVAL;
    }
    PngImage& I = imgs[k];
    I.src = src;
    I.len = P.info.idat_bytes;
    I.raw = raw;
    I.ch = P.info.channels;
    I.pad = 0;
    const int64_t rl = (int64_t)h * (1 + (int64_t)w * I.ch);
    if (rl > INT32_MAX || I.len > INT32_MAX) {
      set_error("udh_png_plan: image %d is too large for one zlib stream of the decoder", k);
      return UDH_EINVAL;
    }
    raw += align_up_png(rl);
    src += I.len;
    *max_row = std::max(*max_row, w * I.ch);
    if (parsed) (*parsed)[k] = P;
  }
  *raw_bytes = raw;
  *idat_bytes = src;
  return UDH_OK;
}

static size_t png_plan_size(int n) { return sizeof(PngPlanHeader) + (size_t)n * sizeof(PngImage); }

}  // namespace udh

using namespace udh;

extern "C" int udh_png_parse(const uint8_t* data, int64_t nbytes, udh_png_info* info) {
  UDH_REQUIRE(info && (data || nbytes == 0) && nbytes >= 0, "udh_png_parse: bad argument");
  PngParsed P;
  const int r = png_parse_impl(data, nbytes, P);
  *info = P.info;
  info->reason = r;
  return UDH_OK;
}

extern "C" size_t udh_png_plan_bytes(const uint8_t* data, const int64_t* offsets, int n, int h, int w, int64_t* idat_bytes) {
  if (!data || !offsets || !idat_bytes || n < 1 || h < 1 || w < 1 || h > 65535 || w > 65535) return 0;
  std::vector<PngImage> imgs;
  int64_t raw, idat;
  int max_row;
  if (png_build_plan(data, offsets, n, h, w, imgs, nullptr, &raw, &idat, &max_row) != UDH_OK) return 0;
  *idat_bytes = idat;
  return png_plan_size(n);
}

extern "C" int udh_png_plan(const uint8_t* data, const int64_t* offsets, int n, int h, int w, void* plan, size_t plan_bytes, uint8_t* idat,
                            int64_t idat_bytes) {
  UDH_REQUIRE(data && offsets && plan && idat, "udh_png_plan: null pointer");
  UDH_REQUIRE(n >= 1 && h >= 1 && w >= 1 && h <= 65535 && w <= 65535, "udh_png_plan: bad dimensions");
  std::vector<PngImage> imgs;
  std::vector<PngParsed> parsed;
  PngPlanHeader hd{};
  int max_row;
  const int rc = png_build_plan(data, offsets, n, h, w, imgs, &parsed, &hd.raw_bytes, &hd.idat_bytes, &max_row);
  if (rc != UDH_OK) return rc;
  const size_t need = png_plan_size(n);
  if (plan_bytes < need || idat_bytes < hd.idat_bytes) {
    set_error("udh_png_plan: plan buffer of %zu bytes (%zu needed), IDAT buffer of %lld bytes (%lld needed)", plan_bytes, need,
              (long long)idat_bytes, (long long)hd.idat_bytes);
    return UDH_EWS;
  }
  for (int k = 0; k < n; ++k) {
    uint8_t* dst = idat + imgs[k].src;
    for (const auto& c : parsed[k].idat) {
      memcpy(dst, data + offsets[k] + c.first, (size_t)c.second);
      dst += c.second;
    }
  }
  hd.magic = kPngMagic;
  hd.n = n;
  hd.h = h;
  hd.w = w;
  hd.max_row = max_row;
  uint8_t* p = static_cast<uint8_t*>(plan);
  memcpy(p, &hd, sizeof(hd));
  memcpy(p + sizeof(hd), imgs.data(), (size_t)n * sizeof(PngImage));
  return UDH_OK;
}

extern "C" size_t udh_png_workspace_bytes(const void* plan_host) {
  if (!plan_host) return 0;
  PngPlanHeader hd;
  memcpy(&hd, plan_host, sizeof(hd));
  if (hd.magic != kPngMagic || hd.n < 1) return 0;
  return (size_t)std::max<int64_t>(hd.raw_bytes, 16);
}

extern "C" int udh_png_decode(const void* plan_host, const void* plan_dev, const uint8_t* idat, uint8_t* out, int32_t* status, int rgb,
                              void* ws, size_t ws_bytes, void* stream) {
  UDH_REQUIRE(plan_host && plan_dev && idat && out && status && ws, "udh_png_decode: null pointer");
  PngPlanHeader hd;
  memcpy(&hd, plan_host, sizeof(hd));
  UDH_REQUIRE(hd.magic == kPngMagic && hd.n >= 1, "udh_png_decode: not a plan made by udh_png_plan");
  const size_t need = udh_png_workspace_bytes(plan_host);
  if (ws_bytes < need) {
    set_error("udh_png_decode: workspace of %zu bytes, %zu needed", ws_bytes, need);
    return UDH_EWS;
  }
  UDH_REQUIRE(((uintptr_t)ws & 15) == 0 && ((uintptr_t)plan_dev & 15) == 0, "udh_png_decode: plan and workspace must be 16-byte aligned");
  const int rowcap = (hd.max_row + 15) / 16 * 16;
  const size_t smem = 2 * (size_t)rowcap;
  if (smem > 200 * 1024) {
    set_error("udh_png_decode: rows of %d samples do not fit the unfilter kernel's shared memory", hd.max_row);
    return UDH_ENOSUP;
  }
  cudaStream_t st = as_stream(stream);
  const PngImage* imgs = reinterpret_cast<const PngImage*>(static_cast<const uint8_t*>(plan_dev) + sizeof(PngPlanHeader));
  uint8_t* raw = static_cast<uint8_t*>(ws);
  UDH_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t) * hd.n, st));
  png_inflate_kernel<<<hd.n, kPngThreads, 0, st>>>(imgs, idat, raw, status, hd.h, hd.w);
  int rc = check_launch("png_inflate");
  if (rc) return rc;
  if (smem > 48 * 1024) UDH_CUDA(cudaFuncSetAttribute(png_unfilter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  png_unfilter_kernel<<<hd.n, kPngThreads, smem, st>>>(imgs, raw, status, out, hd.h, hd.w, rowcap, rgb ? 1 : 0);
  return check_launch("udh_png_decode");
}
