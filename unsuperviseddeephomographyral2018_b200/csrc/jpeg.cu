// Baseline-JPEG decode on the device, bit-identical to libjpeg-turbo's default decompression (what cv2.imread(...,
// IMREAD_COLOR) returns, as RGB): ISLOW integer IDCT, fancy upsampling, jdcolor's fixed-point YCbCr -> RGB.
//   host parser        walks the markers of each file, builds per image the quantisation tables, Huffman fast-lookup
//                      tables (9-bit lookahead + maxcode/valoffset slow path) and a segment list (one entry per restart
//                      interval; one for the whole scan without DRI).  Anything else is rejected with a reason code.
//   jpeg_entropy_kernel one thread per segment, serial within it; the Huffman tables of the CTA's images in shared memory.
//                      Writes the quantised coefficients (int16, natural order) of every block into the workspace.
//   jpeg_sync_kernel / jpeg_scan_kernel / jpeg_write_kernel  the parallel path for long segments (camera frames without
//                      restart markers): self-synchronising Huffman decode, one thread per kJpegSubBytes subsequence
//                      (Weissenberger & Schmidt, ICPP 2018).  Bit-identical to the serial path; a segment whose
//                      subsequences do not synchronise within the round limit goes to jpeg_entropy_kernel instead.
//   jpeg_idct_kernel   one thread per 8x8 block: dequantise + ISLOW IDCT into component sample planes.
//   jpeg_color_kernel  one thread per output pixel: fancy upsampling of the chroma planes + YCbCr -> RGB (gray: Y to R=G=B).
#include <stddef.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace udh {

struct JpegHuff {
  uint16_t look[512];   // 9-bit lookahead: (code length << 8) | symbol, 0 = code longer than 9 bits (or invalid)
  int32_t maxcode[18];  // largest code of length l (-1: none); maxcode[17] is a sentinel
  int32_t valoff[18];   // symbol index of a length-l code = code + valoff[l]
  uint8_t val[256];
};

struct JpegImage {
  JpegHuff huff[4];     // DC table 0, DC table 1, AC table 0, AC table 1
  uint16_t q[3][64];    // per component, natural order
  int32_t ncomp, hmax, vmax, mcus_x, mcus_y, seg0, nseg, pad;
  int32_t hs[3], vs[3], bw[3], bh[3], ch[3], cw[3], dc[3], ac[3];
  int32_t nblk[3];      // bw * bh
  int32_t fancy;        // chroma planes are fancy-upsampled (libjpeg-turbo: downsampled width > 2)
};

struct JpegSeg {
  int64_t begin, end;   // byte range in the concatenated file data (unstuffed and split at RSTn by the decoder)
  int32_t image, mcu0, nmcu, pad;
};

// A segment on the parallel path.  dend: the first byte the serial reader would treat as a marker (or end), so the
// subsequences' readers see no marker and every bit position below 8 * dend is a file bit position.
struct JpegLong {
  int64_t begin, dend;
  int32_t seg, image, sub0, nsub;   // subsequences sub0 .. sub0 + nsub - 1 of the plan's flat list
};

struct JpegPlanHeader {
  uint32_t magic;
  int32_t n, h, w, nseg, nlong;
  int64_t bytes, plane;   // total plan bytes; coefficients per component plane (stride of the workspace planes)
};

// Parallel-path scratch, per subsequence.  A decoder state sits at a block boundary: the bit position of the block's DC
// code (file bits from the start of the concatenated data; -1 = none, the decode before it failed) and its block slot
// within the MCU (luma blocks in raster order, then Cb, then Cr).
struct JpegPState {
  int64_t pos;
  int32_t slot, pad;
};
struct JpegSubRes {        // what one decode of a subsequence found
  int64_t exit_pos;        // state at the first block boundary at or past the next subsequence's start
  int32_t exit_slot;
  int32_t cnt;             // blocks decoded
  int32_t dc[3];           // sum of the DC differences per component
  int32_t err, errblk;     // first error (UDH_JPEG_E_*, 0 = none) and the local block it hit
};
struct JpegSubOut {        // exclusive scan over the segment's subsequences
  int32_t first;           // first block (in decode order within the segment)
  int32_t pred[3];         // DC predictors on entry
};

constexpr int kJpegSubBytes = 256;            // subsequence length; longer than the longest possible block (< 1800 bits)
constexpr int64_t kJpegParallelMin = 1 << 17; // segments this long or longer take the parallel path
constexpr int kJpegMaxRounds = 16;            // synchronisation rounds before a segment goes to the serial path
constexpr int kJpegWarmSubs = 3;              // round 0 decodes this many subsequences before its own (not counted)

// the entropy kernel copies each image's tables into shared memory as int4 words
static_assert(sizeof(JpegHuff) % 16 == 0 && sizeof(JpegImage) % 16 == 0 && offsetof(JpegImage, huff) == 0,
              "JpegImage tables must stay 16-byte aligned in the plan");

constexpr uint32_t kJpegMagic = 0x4a504731u;
constexpr int kJpegImgsPerCta = 8;

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

static inline int64_t jpeg_plane_coefs(int h, int w) { return (int64_t)((h + 15) / 16 * 16) * ((w + 15) / 16 * 16); }

// ---- device: entropy decode ---------------------------------------------------------------------------------------------
struct BitReader {
  const uint8_t* p;
  const uint8_t* end;
  uint64_t acc;   // next bits, MSB first
  int nbits;      // bits in acc
  int fake;       // zero bits appended past the end of the segment's data (the lowest `fake` of the nbits)

  __device__ __forceinline__ void fill() {
    while (nbits <= 56) {
      uint32_t b = 0;
      if (p < end) {
        b = *p++;
        if (b == 0xFF) {
          if (p < end && *p == 0x00) {
            ++p;
          } else {        // a marker: the segment's data ends here
            p = end;
            b = 0;
            fake += 8;
          }
        }
      } else {
        fake += 8;
      }
      acc |= (uint64_t)b << (56 - nbits);
      nbits += 8;
    }
  }
  __device__ __forceinline__ uint32_t peek(int n) const { return (uint32_t)(acc >> (64 - n)); }
  __device__ __forceinline__ bool skip(int n) {   // false when the bits consumed run past the data
    acc <<= n;
    nbits -= n;
    return nbits >= fake;
  }
};

__device__ __forceinline__ int jpeg_extend(uint32_t v, int s) { return (s && v < (1u << (s - 1))) ? (int)v - (1 << s) + 1 : (int)v; }

// BitReader that also knows the file bit position of its next bit: pos counts the bits consumed plus 8 for every
// stuffed 00 passed (marked in `mask` at the last bit of its FF, aligned with acc).
struct PosReader {
  const uint8_t* p;
  const uint8_t* end;
  uint64_t acc, mask;
  int nbits, fake;
  int64_t pos;

  // reader whose next bit is file bit `bitpos` of `data` (bit 0 = MSB of byte 0); bytes at or past `end` read as fake
  __device__ __forceinline__ void init(const uint8_t* data, const uint8_t* e, int64_t bitpos) {
    p = data + (bitpos >> 3);
    end = e;
    if (p > end) p = end;
    acc = mask = 0;
    nbits = fake = 0;
    pos = bitpos & ~(int64_t)7;
    fill();
    skip((int)(bitpos & 7));
  }
  __device__ __forceinline__ void fill() {
    while (nbits <= 56) {
      uint32_t b = 0;
      if (p < end) {
        b = *p++;
        if (b == 0xFF) {
          if (p < end && *p == 0x00) {
            ++p;
            mask |= 1ull << (56 - nbits);
          } else {
            p = end;
            b = 0;
            fake += 8;
          }
        }
      } else {
        fake += 8;
      }
      acc |= (uint64_t)b << (56 - nbits);
      nbits += 8;
    }
  }
  __device__ __forceinline__ uint32_t peek(int n) const { return (uint32_t)(acc >> (64 - n)); }
  __device__ __forceinline__ bool skip(int n) {
    if (n) {
      pos += n + 8 * __popcll(mask >> (64 - n));
      mask <<= n;
    }
    acc <<= n;
    nbits -= n;
    return nbits >= fake;
  }
};

// -1 on an invalid code; otherwise the symbol (the bits are consumed even when they run past the data; the caller checks)
template <class R>
__device__ __forceinline__ int huff_decode(R& br, const JpegHuff& t, bool& ok) {
  const uint32_t e = t.look[br.peek(9)];
  if (e) {
    ok = br.skip(e >> 8);
    return e & 255;
  }
  int l = 10;
  int code = (int)br.peek(10);
  while (l <= 16 && code > t.maxcode[l]) {
    ++l;
    code = (int)br.peek(l);
  }
  if (l > 16) return -1;
  ok = br.skip(l);
  return t.val[(code + t.valoff[l]) & 255];
}

__constant__ uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// Lanes per image (L): each CTA holds the Huffman tables of kJpegImgsPerCta images; thread t serves image t / L and its
// segments t % L, t % L + L, ...  L = 32 gives every image a warp of its own; L = 1 puts the images side by side in one warp.
template <int L>
__global__ void __launch_bounds__(kJpegImgsPerCta * L, 1) jpeg_entropy_kernel(const JpegImage* __restrict__ imgs,
                                                                           const JpegSeg* __restrict__ segs,
                                                                           const uint8_t* __restrict__ data, int16_t* __restrict__ coef,
                                                                           int64_t plane, int32_t* __restrict__ status, int n,
                                                                           const uint8_t* __restrict__ parallel_done) {
  __shared__ __align__(16) JpegHuff tabs[kJpegImgsPerCta][4];
  const int img0 = blockIdx.x * kJpegImgsPerCta;
  const int nimg = min(kJpegImgsPerCta, n - img0);
  {
    constexpr int kWords = (int)(sizeof(JpegHuff) * 4 / 16);
    for (int i = threadIdx.x; i < nimg * kWords; i += blockDim.x) {
      const int k = i / kWords, o = i - k * kWords;
      reinterpret_cast<int4*>(&tabs[k][0])[o] = reinterpret_cast<const int4*>(&imgs[img0 + k].huff[0])[o];
    }
  }
  __syncthreads();
  const int li = threadIdx.x / L, lane = threadIdx.x % L;
  if (li >= nimg) return;
  const int img = img0 + li;
  const JpegImage& im = imgs[img];
  const int ncomp = im.ncomp, mcus_x = im.mcus_x;
  for (int s = lane; s < im.nseg; s += L) {
    if (parallel_done && parallel_done[im.seg0 + s]) continue;   // decoded by the parallel path
    const JpegSeg sg = segs[im.seg0 + s];
    BitReader br{data + sg.begin, data + sg.end, 0, 0, 0};
    int pred0 = 0, pred1 = 0, pred2 = 0;   // DC predictors (scalars: a dynamically indexed array would live in local memory)
    int err = 0;
    for (int m = sg.mcu0; m < sg.mcu0 + sg.nmcu && !err; ++m) {
      const int my = m / mcus_x, mx = m - my * mcus_x;
      for (int c = 0; c < ncomp && !err; ++c) {
        const JpegHuff& dct = tabs[li][im.dc[c]];
        const JpegHuff& act = tabs[li][2 + im.ac[c]];
        const int hs = im.hs[c], vs = im.vs[c], bw = im.bw[c];
        for (int v = 0; v < vs && !err; ++v)
          for (int u = 0; u < hs && !err; ++u) {
            int16_t* blk = coef + ((int64_t)img * 3 + c) * plane + ((int64_t)(my * vs + v) * bw + mx * hs + u) * 64;
#pragma unroll
            for (int k = 0; k < 8; ++k) reinterpret_cast<int4*>(blk)[k] = make_int4(0, 0, 0, 0);
            br.fill();
            bool ok = true;
            int t = huff_decode(br, dct, ok);
            if (t < 0) { err = 2; break; }
            if (t > 15) { err = 2; break; }
            const uint32_t bits = t ? br.peek(t) : 0u;
            ok = br.skip(t) && ok;
            if (!ok) { err = 1; break; }
            const int dc = (c == 0 ? pred0 : c == 1 ? pred1 : pred2) + jpeg_extend(bits, t);
            if (c == 0) pred0 = dc; else if (c == 1) pred1 = dc; else pred2 = dc;
            blk[0] = (int16_t)dc;
            for (int k = 1; k < 64;) {
              br.fill();
              const int rs = huff_decode(br, act, ok);
              if (rs < 0) { err = 2; break; }
              if (!ok) { err = 1; break; }
              const int r = rs >> 4, sz = rs & 15;
              if (sz) {
                k += r;
                if (k > 63) { err = 3; break; }
                const uint32_t b = br.peek(sz);
                if (!br.skip(sz)) { err = 1; break; }
                blk[kZigzag[k]] = (int16_t)jpeg_extend(b, sz);
                ++k;
              } else if (r == 15) {
                k += 16;
              } else {
                break;
              }
            }
          }
      }
    }
    if (err) atomicCAS(&status[img], 0, err);
  }
}

// ---- device: parallel entropy decode of long segments -----------------------------------------------------------------
// 1. jpeg_sync_kernel, round 0: thread i decodes from the start of subsequence i - kJpegWarmSubs (byte begin +
//    k * kJpegSubBytes, one byte later when that byte is the 00 of a stuffed FF 00; block slot 0) up to its own
//    subsequence and takes the block boundary it reaches there as its start; threads i <= kJpegWarmSubs thereby start in
//    the true state.  A decode that begins at a guessed bit position soon meets the true codeword boundaries, but it
//    needs the true block slot too (luma and chroma tables differ), which one subsequence is often too short to find.
//    Each thread then decodes whole blocks until the first block boundary at or past the next subsequence's start and
//    records that exit state, its block count, its DC difference sums and its first error.
// 2. Rounds 1..R: subsequence i restarts from i-1's exit state (its own assumed start when i-1 failed); a thread whose
//    start did not change copies its previous result.  A round in which no exit state changes proves every start state
//    true by induction from subsequence 0.  A segment still changing after R rounds goes to the serial kernel.
// 3. jpeg_scan_kernel: exclusive scan of the block counts and DC sums -> each subsequence's first block and its DC
//    predictors; the first error before the segment's last block becomes the image's status (as the serial path would).
// 4. jpeg_write_kernel: each subsequence decodes again from its synchronised start and stores its blocks.
// Errors met before synchronisation are speculative and never reach `status`.

struct JpegSlotMap {   // block slot -> component and block offset within the MCU
  int bpm, ny, hs0;
  __device__ __forceinline__ JpegSlotMap(const JpegImage& im)
      : bpm(im.ncomp == 1 ? 1 : im.hs[0] * im.vs[0] + 2), ny(im.hs[0] * im.vs[0]), hs0(im.hs[0]) {}
  __device__ __forceinline__ int comp(int slot) const { return slot < ny ? 0 : slot - ny + 1; }
};

// One block as jpeg_entropy_kernel decodes it (same checks, same order, same codes); blk == nullptr: count only.
// Returns 0 or the UDH_JPEG_E_* code; *dcdiff = the DC difference.
__device__ __forceinline__ int jpeg_block(PosReader& br, const JpegHuff& dct, const JpegHuff& act, int* dcdiff, int16_t* blk) {
  if (blk) {
#pragma unroll
    for (int k = 0; k < 8; ++k) reinterpret_cast<int4*>(blk)[k] = make_int4(0, 0, 0, 0);
  }
  br.fill();
  bool ok = true;
  const int t = huff_decode(br, dct, ok);
  if (t < 0 || t > 15) return 2;
  const uint32_t bits = t ? br.peek(t) : 0u;
  ok = br.skip(t) && ok;
  if (!ok) return 1;
  *dcdiff = jpeg_extend(bits, t);
  for (int k = 1; k < 64;) {
    br.fill();
    const int rs = huff_decode(br, act, ok);
    if (rs < 0) return 2;
    if (!ok) return 1;
    const int r = rs >> 4, sz = rs & 15;
    if (sz) {
      k += r;
      if (k > 63) return 3;
      const uint32_t b = br.peek(sz);
      if (!br.skip(sz)) return 1;
      if (blk) blk[kZigzag[k]] = (int16_t)jpeg_extend(b, sz);
      ++k;
    } else if (r == 15) {
      k += 16;
    } else {
      break;
    }
  }
  return 0;
}

// first byte of subsequence i (the byte after a stuffed pair's FF rather than its 00)
__device__ __forceinline__ int64_t jpeg_sub_start(const JpegLong& L, const uint8_t* data, int i) {
  int64_t b = L.begin + (int64_t)i * kJpegSubBytes;
  if (i > 0 && b < L.dend && data[b - 1] == 0xFF) ++b;
  return b;
}

__device__ __forceinline__ void jpeg_load_tables(JpegHuff (&tabs)[4], const JpegImage& im) {
  constexpr int kWords = (int)(sizeof(JpegHuff) * 4 / 16);
  for (int i = threadIdx.x; i < kWords; i += blockDim.x)
    reinterpret_cast<int4*>(&tabs[0])[i] = reinterpret_cast<const int4*>(&im.huff[0])[i];
  __syncthreads();
}

// grid (subsequence chunks, long segments); round 0 seeds every state, round r >= 1 synchronises
__global__ void __launch_bounds__(128) jpeg_sync_kernel(const JpegImage* __restrict__ imgs, const JpegSeg* __restrict__ segs,
                                                        const JpegLong* __restrict__ longs, const uint8_t* __restrict__ data,
                                                        JpegSubRes* __restrict__ res, JpegPState* __restrict__ used,
                                                        int32_t* __restrict__ changed, int64_t nsub_all, int round) {
  const JpegLong L = longs[blockIdx.y];
  if (blockIdx.x * blockDim.x >= L.nsub) return;
  int32_t* chg = changed + (int64_t)blockIdx.y * (kJpegMaxRounds + 1);
  if (round >= 2 && chg[round - 1] == 0) return;   // converged in an earlier round
  __shared__ __align__(16) JpegHuff tabs[4];
  const JpegImage& im = imgs[L.image];
  jpeg_load_tables(tabs, im);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L.nsub) return;
  const int64_t g = L.sub0 + i;
  const JpegSubRes* prev = res + (int64_t)((round + 1) & 1) * nsub_all;
  JpegSubRes* cur = res + (int64_t)(round & 1) * nsub_all;
  const JpegSeg sg = segs[L.seg];
  const JpegSlotMap sm(im);
  const int64_t total = (int64_t)sg.nmcu * sm.bpm;
  JpegPState st{8 * jpeg_sub_start(L, data, i), 0, 0};
  PosReader br;
  bool positioned = false;
  if (round == 0 && i > 0) {
    br.init(data, data + L.dend, 8 * jpeg_sub_start(L, data, max(0, i - kJpegWarmSubs)));
    int slot = 0, werr = 0, d = 0;
    for (int64_t n = 0; br.pos < st.pos && n < total && !werr; ++n) {
      werr = jpeg_block(br, tabs[im.dc[sm.comp(slot)]], tabs[2 + im.ac[sm.comp(slot)]], &d, nullptr);
      if (++slot == sm.bpm) slot = 0;
    }
    if (!werr) {
      st = JpegPState{br.pos, slot, 0};
      positioned = true;
    }
  }
  if (round > 0 && i > 0 && prev[g - 1].exit_pos >= 0) st = JpegPState{prev[g - 1].exit_pos, prev[g - 1].exit_slot, 0};
  if (round > 0 && st.pos == used[g].pos && st.slot == used[g].slot) {
    cur[g] = prev[g];
    return;
  }
  used[g] = st;
  const int64_t limit = i + 1 < L.nsub ? 8 * jpeg_sub_start(L, data, i + 1) : INT64_MAX;
  if (!positioned) br.init(data, data + L.dend, st.pos);
  int slot = st.slot, cnt = 0, err = 0, dc[3] = {0, 0, 0};
  while (br.pos < limit && cnt < total) {
    const int c = sm.comp(slot);
    int d = 0;
    err = jpeg_block(br, tabs[im.dc[c]], tabs[2 + im.ac[c]], &d, nullptr);
    if (err) break;
    dc[0] += c == 0 ? d : 0; dc[1] += c == 1 ? d : 0; dc[2] += c == 2 ? d : 0;
    ++cnt;
    if (++slot == sm.bpm) slot = 0;
  }
  JpegSubRes r;
  r.exit_pos = err ? -1 : br.pos;
  r.exit_slot = err ? 0 : slot;
  r.cnt = cnt;
  r.dc[0] = dc[0]; r.dc[1] = dc[1]; r.dc[2] = dc[2];
  r.err = err;
  r.errblk = cnt;
  cur[g] = r;
  if (round > 0 && (r.exit_pos != prev[g].exit_pos || r.exit_slot != prev[g].exit_slot)) chg[round] = 1;
}

// inclusive warp scan of four ints
__device__ __forceinline__ void warp_scan4(int4& v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int a = __shfl_up_sync(0xffffffffu, v.x, o), b = __shfl_up_sync(0xffffffffu, v.y, o);
    const int c = __shfl_up_sync(0xffffffffu, v.z, o), d = __shfl_up_sync(0xffffffffu, v.w, o);
    if (lane >= o) { v.x += a; v.y += b; v.z += c; v.w += d; }
  }
}

// one CTA of 1024 threads per long segment
__global__ void __launch_bounds__(1024) jpeg_scan_kernel(const JpegImage* __restrict__ imgs, const JpegSeg* __restrict__ segs,
                                                         const JpegLong* __restrict__ longs, const JpegSubRes* __restrict__ res,
                                                         const int32_t* __restrict__ changed, JpegSubOut* __restrict__ outp,
                                                         uint8_t* __restrict__ parallel_done, int32_t* __restrict__ status,
                                                         int64_t nsub_all, int rounds) {
  const JpegLong L = longs[blockIdx.x];
  const int32_t* chg = changed + (int64_t)blockIdx.x * (kJpegMaxRounds + 1);
  int conv = 0;
  for (int r = 1; r <= rounds && !conv; ++r)
    if (chg[r] == 0) conv = r;
  if (!conv) return;   // not synchronised: the serial kernel decodes this segment
  const JpegSubRes* rs = res + (int64_t)(conv & 1) * nsub_all + L.sub0;
  const int64_t total = (int64_t)segs[L.seg].nmcu * JpegSlotMap(imgs[L.image]).bpm;
  __shared__ int4 wsum[32];
  __shared__ int4 carry;
  __shared__ int first_err;
  if (threadIdx.x == 0) { carry = make_int4(0, 0, 0, 0); first_err = INT32_MAX; }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int base = 0; base < L.nsub; base += blockDim.x) {
    const int i = base + threadIdx.x;
    int4 v = make_int4(0, 0, 0, 0);
    if (i < L.nsub) v = make_int4(rs[i].cnt, rs[i].dc[0], rs[i].dc[1], rs[i].dc[2]);
    const int4 own = v;
    warp_scan4(v);
    if (lane == 31) wsum[warp] = v;
    __syncthreads();
    if (warp == 0) {
      int4 w = wsum[lane];
      warp_scan4(w);
      wsum[lane] = w;
    }
    __syncthreads();
    const int4 c0 = carry;
    int4 ex = make_int4(c0.x + v.x - own.x, c0.y + v.y - own.y, c0.z + v.z - own.z, c0.w + v.w - own.w);
    if (warp > 0) { const int4 p = wsum[warp - 1]; ex.x += p.x; ex.y += p.y; ex.z += p.z; ex.w += p.w; }
    if (i < L.nsub) {
      JpegSubOut o;
      o.first = ex.x;
      o.pred[0] = ex.y; o.pred[1] = ex.z; o.pred[2] = ex.w;
      outp[L.sub0 + i] = o;
      if (rs[i].err && (int64_t)ex.x + rs[i].errblk < total) atomicMin(&first_err, i);
    }
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) {
      const int4 t = wsum[31];
      carry = make_int4(c0.x + t.x, c0.y + t.y, c0.z + t.z, c0.w + t.w);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    parallel_done[L.seg] = 1;
    if (first_err != INT32_MAX) atomicCAS(&status[L.image], 0, rs[first_err].err);
  }
}

__global__ void __launch_bounds__(128) jpeg_write_kernel(const JpegImage* __restrict__ imgs, const JpegSeg* __restrict__ segs,
                                                         const JpegLong* __restrict__ longs, const uint8_t* __restrict__ data,
                                                         const JpegPState* __restrict__ used, const JpegSubOut* __restrict__ outp,
                                                         const uint8_t* __restrict__ parallel_done, int16_t* __restrict__ coef,
                                                         int64_t plane) {
  const JpegLong L = longs[blockIdx.y];
  if (blockIdx.x * blockDim.x >= L.nsub || !parallel_done[L.seg]) return;
  __shared__ __align__(16) JpegHuff tabs[4];
  const JpegImage& im = imgs[L.image];
  jpeg_load_tables(tabs, im);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L.nsub) return;
  const int64_t g = L.sub0 + i;
  const JpegSeg sg = segs[L.seg];
  const JpegSlotMap sm(im);
  const int64_t total = (int64_t)sg.nmcu * sm.bpm;
  const JpegSubOut o = outp[g];
  if (o.first >= total) return;
  const int64_t limit = i + 1 < L.nsub ? 8 * jpeg_sub_start(L, data, i + 1) : INT64_MAX;
  PosReader br;
  br.init(data, data + L.dend, used[g].pos);
  int pred0 = o.pred[0], pred1 = o.pred[1], pred2 = o.pred[2];
  const int mcus_x = im.mcus_x;
  int m = sg.mcu0 + o.first / sm.bpm, slot = o.first % sm.bpm;
  for (int64_t b = o.first; b < total && br.pos < limit; ++b) {
    const int c = sm.comp(slot);
    const int my = m / mcus_x, mx = m - my * mcus_x;
    const int v = c ? 0 : slot / sm.hs0, u = c ? 0 : slot - v * sm.hs0;
    int16_t* blk = coef + ((int64_t)L.image * 3 + c) * plane + ((int64_t)(my * im.vs[c] + v) * im.bw[c] + mx * im.hs[c] + u) * 64;
    int d = 0;
    if (jpeg_block(br, tabs[im.dc[c]], tabs[2 + im.ac[c]], &d, blk)) return;   // reported by jpeg_scan_kernel
    const int dc = (c == 0 ? pred0 : c == 1 ? pred1 : pred2) + d;
    if (c == 0) pred0 = dc; else if (c == 1) pred1 = dc; else pred2 = dc;
    blk[0] = (int16_t)dc;
    if (++slot == sm.bpm) { slot = 0; ++m; }
  }
}

// ---- device: dequantise + ISLOW IDCT ---------------------------------------------------------------------------------
// jidctint.c's scheme: CONST_BITS 13, PASS1_BITS 2; columns first, rows second; outputs through the sample range-limit
// table, which wraps the descaled value to 10 bits (RANGE_MASK) before clamping 128 + v to 0..255.
constexpr int kF0298 = 2446, kF0390 = 3196, kF0541 = 4433, kF0765 = 6270, kF0899 = 7373, kF1175 = 9633, kF1501 = 12299,
              kF1847 = 15137, kF1961 = 16069, kF2053 = 16819, kF2562 = 20995, kF3072 = 25172;

template <int SHIFT>
__device__ __forceinline__ void idct_1d(const int x0, const int x1, const int x2, const int x3, const int x4, const int x5,
                                        const int x6, const int x7, int (&o)[8]) {
  int z1 = (x2 + x6) * kF0541;
  const int tmp2 = z1 - x6 * kF1847, tmp3 = z1 + x2 * kF0765;
  const int tmp0 = (x0 + x4) * (1 << 13), tmp1 = (x0 - x4) * (1 << 13);
  const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int t0 = x7, t1 = x5, t2 = x3, t3 = x1;
  z1 = t0 + t3;
  int z2 = t1 + t2, z3 = t0 + t2, z4 = t1 + t3;
  const int z5 = (z3 + z4) * kF1175;
  t0 *= kF0298; t1 *= kF2053; t2 *= kF3072; t3 *= kF1501;
  z1 *= -kF0899; z2 *= -kF2562; z3 = z3 * -kF1961 + z5; z4 = z4 * -kF0390 + z5;
  t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;
  constexpr int R = 1 << (SHIFT - 1);
  o[0] = (t10 + t3 + R) >> SHIFT; o[7] = (t10 - t3 + R) >> SHIFT;
  o[1] = (t11 + t2 + R) >> SHIFT; o[6] = (t11 - t2 + R) >> SHIFT;
  o[2] = (t12 + t1 + R) >> SHIFT; o[5] = (t12 - t1 + R) >> SHIFT;
  o[3] = (t13 + t0 + R) >> SHIFT; o[4] = (t13 - t0 + R) >> SHIFT;
}

__device__ __forceinline__ uint32_t idct_limit(int v) {
  v = ((v & 1023) ^ 512) - 512;
  return (uint32_t)min(max(v + 128, 0), 255);
}

__global__ void __launch_bounds__(128) jpeg_idct_kernel(const JpegImage* __restrict__ imgs, const int16_t* __restrict__ coef,
                                                        uint8_t* __restrict__ samples, int64_t plane) {
  const int img = blockIdx.y;
  const JpegImage& im = imgs[img];
  int b = blockIdx.x * blockDim.x + threadIdx.x, c = 0;
  while (c < im.ncomp && b >= im.nblk[c]) b -= im.nblk[c++];
  if (c >= im.ncomp) return;
  const int16_t* src = coef + ((int64_t)img * 3 + c) * plane + (int64_t)b * 64;
  const uint16_t* q = im.q[c];
  int ws[64];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int4 v = __ldg(reinterpret_cast<const int4*>(src) + k);
    const int16_t* s = reinterpret_cast<const int16_t*>(&v);
#pragma unroll
    for (int j = 0; j < 8; ++j) ws[k * 8 + j] = (int)s[j] * (int)q[k * 8 + j];
  }
#pragma unroll
  for (int x = 0; x < 8; ++x) {          // pass 1: columns
    int o[8];
    idct_1d<11>(ws[x], ws[8 + x], ws[16 + x], ws[24 + x], ws[32 + x], ws[40 + x], ws[48 + x], ws[56 + x], o);
#pragma unroll
    for (int y = 0; y < 8; ++y) ws[y * 8 + x] = o[y];
  }
  const int by = b / im.bw[c], bx = b - by * im.bw[c];
  const int pw = im.bw[c] * 8;
  uint8_t* dst = samples + ((int64_t)img * 3 + c) * plane + (int64_t)by * 8 * pw + bx * 8;
#pragma unroll
  for (int y = 0; y < 8; ++y) {          // pass 2: rows
    int o[8];
    idct_1d<18>(ws[y * 8], ws[y * 8 + 1], ws[y * 8 + 2], ws[y * 8 + 3], ws[y * 8 + 4], ws[y * 8 + 5], ws[y * 8 + 6], ws[y * 8 + 7], o);
    uint2 r;
    r.x = idct_limit(o[0]) | idct_limit(o[1]) << 8 | idct_limit(o[2]) << 16 | idct_limit(o[3]) << 24;
    r.y = idct_limit(o[4]) | idct_limit(o[5]) << 8 | idct_limit(o[6]) << 16 | idct_limit(o[7]) << 24;
    *reinterpret_cast<uint2*>(dst + (int64_t)y * pw) = r;
  }
}

// ---- device: upsampling + colour conversion ------------------------------------------------------------------------
// jdsample.c: h2v1 = 3:1 horizontal triangle, bias +1 / +2 (even / odd output); h2v2 = the same on 3:1 column sums, bias
// +8 / +7; the outermost sample is replicated at every edge.  Planes <= 2 samples wide are replicated, not filtered.
__device__ __forceinline__ int chroma_at(const uint8_t* p, int pw, int ch, int cw, int hf, int vf, bool fancy, int y, int x) {
  const int r = vf == 2 ? y >> 1 : y, k = hf == 2 ? x >> 1 : x;
  if (!fancy || (hf == 1 && vf == 1)) return p[(int64_t)r * pw + k];
  const int kn = (x & 1) ? min(k + 1, cw - 1) : max(k - 1, 0);
  if (vf == 1) {
    const int a = p[(int64_t)r * pw + k], b = p[(int64_t)r * pw + kn];
    return (3 * a + b + ((x & 1) ? 2 : 1)) >> 2;
  }
  const int rn = (y & 1) ? min(r + 1, ch - 1) : max(r - 1, 0);
  const uint8_t* p0 = p + (int64_t)r * pw;
  const uint8_t* p1 = p + (int64_t)rn * pw;
  const int c0 = 3 * p0[k] + p1[k], c1 = 3 * p0[kn] + p1[kn];
  return (3 * c0 + c1 + ((x & 1) ? 7 : 8)) >> 4;
}

__global__ void __launch_bounds__(256) jpeg_color_kernel(const JpegImage* __restrict__ imgs, const uint8_t* __restrict__ samples,
                                                         int64_t plane, uint8_t* __restrict__ out, int h, int w) {
  const int img = blockIdx.y;
  const JpegImage& im = imgs[img];
  const int npx = h * w;
  const uint8_t* Y = samples + (int64_t)img * 3 * plane;
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < npx; o += gridDim.x * blockDim.x) {
    const int y = o / w, x = o - y * w;
    const int yy = Y[(int64_t)y * im.bw[0] * 8 + x];
    uint8_t* dst = out + ((int64_t)img * npx + o) * 3;
    if (im.ncomp == 1) {
      dst[0] = dst[1] = dst[2] = (uint8_t)yy;
      continue;
    }
    const int hf = im.hmax / im.hs[1], vf = im.vmax / im.vs[1];
    const int cb = chroma_at(Y + plane, im.bw[1] * 8, im.ch[1], im.cw[1], hf, vf, im.fancy, y, x) - 128;
    const int cr = chroma_at(Y + 2 * plane, im.bw[2] * 8, im.ch[2], im.cw[2], hf, vf, im.fancy, y, x) - 128;
    // jdcolor.c build_ycc_rgb_table: FIX(x) = (int)(x * 65536 + 0.5), ONE_HALF = 1 << 15
    const int r = yy + ((91881 * cr + 32768) >> 16);
    const int g = yy + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
    const int b = yy + ((116130 * cb + 32768) >> 16);
    dst[0] = (uint8_t)min(max(r, 0), 255);
    dst[1] = (uint8_t)min(max(g, 0), 255);
    dst[2] = (uint8_t)min(max(b, 0), 255);
  }
}

// ---- host: parser ----------------------------------------------------------------------------------------------------
struct JpegParsed {
  udh_jpeg_info info;
  JpegImage img;
  int64_t scan_begin;   // first entropy-coded byte (file-relative)
};

static int jpeg_u16(const uint8_t* d) { return (d[0] << 8) | d[1]; }

// jdhuff.c's checks (jpeg_make_d_derived_tbl): at most 256 symbols, DC symbols <= 15, and every code fits its length
// without being all ones.  They run before any lookahead entry is written, so a malformed table never writes past look[].
static bool build_huff(const uint8_t* counts, const uint8_t* vals, int nvals, bool dc, JpegHuff& t) {
  memset(&t, 0, sizeof(t));
  if (nvals > 256) return false;
  for (int i = 0; dc && i < nvals; ++i)
    if (vals[i] > 15) return false;
  for (int l = 1, code = 0; l <= 16; ++l) {
    code += counts[l - 1];
    if (code >= (1 << l)) return false;   // over-subscribed lengths, or an all-ones code
    code <<= 1;
  }
  memcpy(t.val, vals, nvals);
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    t.valoff[l] = k - code;
    for (int i = 0; i < counts[l - 1]; ++i, ++k, ++code) {
      if (l <= 9) {
        const int first = code << (9 - l), num = 1 << (9 - l);
        for (int j = 0; j < num; ++j) t.look[first + j] = (uint16_t)(l << 8 | vals[k]);
      }
    }
    t.maxcode[l] = counts[l - 1] ? code - 1 : -1;
    code <<= 1;
  }
  t.maxcode[17] = 0x7fffffff;
  return true;
}

// EXIF orientation (TIFF tag 0x0112 of IFD0) of an APP1 payload, 1 when absent or unreadable
static int exif_orientation(const uint8_t* s, int n) {
  if (n < 14 || memcmp(s, "Exif\0\0", 6) != 0) return 1;
  const uint8_t* t = s + 6;
  const int tn = n - 6;
  const bool le = t[0] == 'I' && t[1] == 'I';
  if (!le && !(t[0] == 'M' && t[1] == 'M')) return 1;
  auto rd16 = [&](int o) -> int { return o + 2 > tn ? -1 : (le ? (t[o] | t[o + 1] << 8) : (t[o] << 8 | t[o + 1])); };
  auto rd32 = [&](int o) -> int64_t {
    if (o + 4 > tn) return -1;
    return le ? ((int64_t)t[o] | (int64_t)t[o + 1] << 8 | (int64_t)t[o + 2] << 16 | (int64_t)t[o + 3] << 24)
              : ((int64_t)t[o] << 24 | (int64_t)t[o + 1] << 16 | (int64_t)t[o + 2] << 8 | (int64_t)t[o + 3]);
  };
  const int64_t ifd = rd32(4);
  if (ifd < 8 || ifd + 2 > tn) return 1;
  const int cnt = rd16((int)ifd);
  for (int i = 0; i < cnt; ++i) {
    const int e = (int)ifd + 2 + 12 * i;
    if (e + 12 > tn) break;
    if (rd16(e) == 0x0112) return rd16(e + 8);
  }
  return 1;
}

static int jpeg_parse_impl(const uint8_t* d, int64_t n, JpegParsed& P) {
  memset(&P, 0, sizeof(P));
  udh_jpeg_info& I = P.info;
  JpegImage& M = P.img;
  if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) return UDH_JPEG_R_NOT_JPEG;
  bool have_q[4] = {}, have_dc[2] = {}, have_ac[2] = {}, frame = false, jfif = false, adobe = false;
  int adobe_transform = -1, orientation = 1;
  uint16_t qt[4][64];
  int cid[3] = {0, 0, 0}, tq[3] = {0, 0, 0};
  int64_t i = 2;
  for (;;) {
    while (i + 1 < n && d[i] == 0xFF && d[i + 1] == 0xFF) ++i;
    if (i + 4 > n || d[i] != 0xFF) return UDH_JPEG_R_TRUNCATED;
    const int m = d[i + 1];
    if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) return UDH_JPEG_R_TRUNCATED;   // no scan before
    const int len = jpeg_u16(d + i + 2);
    if (len < 2 || i + 2 + len > n) return UDH_JPEG_R_TRUNCATED;
    const uint8_t* s = d + i + 4;
    const int sl = len - 2;
    if (m == 0xC0 || m == 0xC1) {
      if (frame || sl < 6) return UDH_JPEG_R_TRUNCATED;
      if (s[0] != 8) return UDH_JPEG_R_PRECISION;
      I.height = jpeg_u16(s + 1);
      I.width = jpeg_u16(s + 3);
      I.components = s[5];
      if (sl < 6 + 3 * s[5]) return UDH_JPEG_R_TRUNCATED;
      if (I.width == 0 || I.height == 0) return UDH_JPEG_R_TRUNCATED;
      if (I.components != 1 && I.components != 3) return UDH_JPEG_R_COMPONENTS;
      for (int c = 0; c < I.components; ++c) {
        cid[c] = s[6 + 3 * c];
        I.h_samp[c] = s[7 + 3 * c] >> 4;
        I.v_samp[c] = s[7 + 3 * c] & 15;
        tq[c] = s[8 + 3 * c];
        if (I.h_samp[c] < 1 || I.h_samp[c] > 4 || I.v_samp[c] < 1 || I.v_samp[c] > 4 || tq[c] > 3) return UDH_JPEG_R_TRUNCATED;
      }
      frame = true;
    } else if (m == 0xC2 || m == 0xC3 || (m >= 0xC5 && m <= 0xCF && m != 0xC8 && m != 0xCC) || m == 0xCC) {
      return UDH_JPEG_R_NOT_BASELINE;   // progressive, lossless, hierarchical or arithmetic-coded
    } else if (m == 0xDB) {
      for (int j = 0; j < sl;) {
        const int pq = s[j] >> 4, t = s[j] & 15, sz = pq ? 128 : 64;
        if (t > 3 || pq > 1 || j + 1 + sz > sl) return UDH_JPEG_R_TRUNCATED;
        for (int k = 0; k < 64; ++k) {
          static const uint8_t zz[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                         41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                         30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
          qt[t][zz[k]] = pq ? (uint16_t)jpeg_u16(s + j + 1 + 2 * k) : s[j + 1 + k];
        }
        have_q[t] = true;
        j += 1 + sz;
      }
    } else if (m == 0xC4) {
      for (int j = 0; j < sl;) {
        if (j + 17 > sl) return UDH_JPEG_R_TRUNCATED;
        const int tc = s[j] >> 4, th = s[j] & 15;
        int nv = 0;
        for (int k = 0; k < 16; ++k) nv += s[j + 1 + k];
        if (tc > 1 || th > 1 || j + 17 + nv > sl) return UDH_JPEG_R_TRUNCATED;
        if (!build_huff(s + j + 1, s + j + 17, nv, tc == 0, M.huff[tc * 2 + th])) return UDH_JPEG_R_TRUNCATED;
        (tc ? have_ac : have_dc)[th] = true;
        j += 17 + nv;
      }
    } else if (m == 0xDD) {
      if (sl < 2) return UDH_JPEG_R_TRUNCATED;
      I.restart_interval = jpeg_u16(s);
    } else if (m == 0xE0) {
      if (sl >= 5 && memcmp(s, "JFIF\0", 5) == 0) jfif = true;
    } else if (m == 0xE1) {
      const int o = exif_orientation(s, sl);
      if (o != 1) orientation = o;
    } else if (m == 0xEE) {
      if (sl >= 12 && memcmp(s, "Adobe", 5) == 0) {
        adobe = true;
        adobe_transform = s[11];
      }
    } else if (m == 0xDA) {
      if (!frame || sl < 1) return UDH_JPEG_R_TRUNCATED;
      const int ns = s[0];
      if (sl < 4 + 2 * ns) return UDH_JPEG_R_TRUNCATED;
      if (ns != I.components) return UDH_JPEG_R_MULTI_SCAN;
      for (int k = 0; k < ns; ++k) {
        if (s[1 + 2 * k] != cid[k]) return UDH_JPEG_R_MULTI_SCAN;   // scan order = frame order
        M.dc[k] = s[2 + 2 * k] >> 4;
        M.ac[k] = s[2 + 2 * k] & 15;
        if (M.dc[k] > 1 || M.ac[k] > 1 || !have_dc[M.dc[k]] || !have_ac[M.ac[k]] || !have_q[tq[k]]) return UDH_JPEG_R_TRUNCATED;
      }
      if (s[1 + 2 * ns] != 0 || s[2 + 2 * ns] != 63 || s[3 + 2 * ns] != 0) return UDH_JPEG_R_TRUNCATED;   // Ss, Se, Ah/Al
      P.scan_begin = i + 2 + len;
      break;
    }
    i += 2 + len;
  }
  // libjpeg's colour-space guess for 3 components (jdapimin.c default_decompress_parms)
  if (I.components == 3 && !jfif) {
    if (adobe ? adobe_transform == 0 : (cid[0] == 'R' && cid[1] == 'G' && cid[2] == 'B')) return UDH_JPEG_R_RGB;
  }
  if (orientation != 1) return UDH_JPEG_R_ORIENTATION;
  M.ncomp = I.components;
  if (I.components == 1) {
    M.hs[0] = M.vs[0] = M.hmax = M.vmax = 1;
  } else {
    const int h0 = I.h_samp[0], v0 = I.v_samp[0];
    for (int c = 1; c < 3; ++c)
      if (I.h_samp[c] != 1 || I.v_samp[c] != 1) return UDH_JPEG_R_SAMPLING_H;
    if (h0 > 2) return UDH_JPEG_R_SAMPLING_H;
    if (v0 > h0) return UDH_JPEG_R_SAMPLING_V;
    for (int c = 0; c < 3; ++c) { M.hs[c] = I.h_samp[c]; M.vs[c] = I.v_samp[c]; }
    M.hmax = h0; M.vmax = v0;
  }
  const int W = I.width, H = I.height;
  M.mcus_x = (W + 8 * M.hmax - 1) / (8 * M.hmax);
  M.mcus_y = (H + 8 * M.vmax - 1) / (8 * M.vmax);
  for (int c = 0; c < M.ncomp; ++c) {
    M.bw[c] = M.mcus_x * M.hs[c];
    M.bh[c] = M.mcus_y * M.vs[c];
    M.nblk[c] = M.bw[c] * M.bh[c];
    M.cw[c] = (W * M.hs[c] + M.hmax - 1) / M.hmax;
    M.ch[c] = (H * M.vs[c] + M.vmax - 1) / M.vmax;
    memcpy(M.q[c], qt[tq[c]], sizeof(M.q[c]));
  }
  M.fancy = M.ncomp == 3 && M.cw[1] > 2;
  return UDH_JPEG_R_OK;
}

// Segments of one parsed file: [begin, end) file-relative; RSTn split only when the file has a restart interval
static void jpeg_segments(const uint8_t* d, int64_t n, const JpegParsed& P, std::vector<JpegSeg>& out, int64_t base, int image) {
  const int nmcu = P.img.mcus_x * P.img.mcus_y;
  const int ri = P.info.restart_interval ? P.info.restart_interval : nmcu;
  const int nseg = (nmcu + ri - 1) / ri;
  int64_t pos = P.scan_begin;
  for (int s = 0; s < nseg; ++s) {
    JpegSeg g{};
    g.image = image;
    g.mcu0 = s * ri;
    g.nmcu = nmcu - s * ri < ri ? nmcu - s * ri : ri;
    g.begin = base + pos;
    int64_t e = n;
    if (s + 1 < nseg) {
      for (int64_t j = pos; j + 1 < n; ++j) {
        const uint8_t* f = static_cast<const uint8_t*>(memchr(d + j, 0xFF, (size_t)(n - 1 - j)));
        if (!f) break;
        j = f - d;
        if (d[j + 1] >= 0xD0 && d[j + 1] <= 0xD7) { e = j; break; }
      }
    }
    g.end = base + e;
    out.push_back(g);
    pos = e < n ? e + 2 : n;
  }
}

// -1: segments of kJpegParallelMin bytes or more take the parallel path; 0: none does; 1: every segment does
static int g_jpeg_parallel = -1;

// The serial reader's end of a segment's data: the first FF not followed by a stuffed 00 (a marker), or end.
static int64_t jpeg_data_end(const uint8_t* d, int64_t begin, int64_t end) {
  for (int64_t j = begin; j < end;) {
    const uint8_t* f = static_cast<const uint8_t*>(memchr(d + j, 0xFF, (size_t)(end - j)));
    if (!f) break;
    j = f - d;
    if (j + 1 < end && d[j + 1] == 0x00) j += 2;
    else return j;
  }
  return end;
}

static void jpeg_long_segments(const uint8_t* data, const std::vector<JpegSeg>& segs, std::vector<JpegLong>& longs) {
  longs.clear();
  int64_t sub = 0;
  for (size_t s = 0; s < segs.size(); ++s) {
    const JpegSeg& g = segs[s];
    if (!(g_jpeg_parallel == 1 || (g_jpeg_parallel < 0 && g.end - g.begin >= kJpegParallelMin))) continue;
    JpegLong L{};
    L.begin = g.begin;
    L.dend = jpeg_data_end(data, g.begin, g.end);
    L.seg = (int)s;
    L.image = g.image;
    L.sub0 = (int)sub;
    L.nsub = (int)std::max<int64_t>(1, (L.dend - L.begin + kJpegSubBytes - 1) / kJpegSubBytes);
    sub += L.nsub;
    longs.push_back(L);
  }
}

static int jpeg_build_plan(const uint8_t* data, const int64_t* offsets, int n, int h, int w, std::vector<JpegImage>& imgs,
                           std::vector<JpegSeg>& segs, std::vector<JpegLong>& longs) {
  imgs.resize(n);
  segs.clear();
  longs.clear();
  JpegParsed P;
  for (int k = 0; k < n; ++k) {
    const int64_t b = offsets[k], len = offsets[k + 1] - offsets[k];
    if (len < 0) {
      set_error("udh_jpeg_plan: offsets must not decrease (image %d)", k);
      return UDH_EINVAL;
    }
    const int r = jpeg_parse_impl(data + b, len, P);
    if (r != UDH_JPEG_R_OK) {
      set_error("udh_jpeg_plan: image %d is not supported (reason %d)", k, r);
      return UDH_ENOSUP;
    }
    if (P.info.height != h || P.info.width != w) {
      set_error("udh_jpeg_plan: image %d is %dx%d, the plan is for %dx%d", k, P.info.height, P.info.width, h, w);
      return UDH_EINVAL;
    }
    P.img.seg0 = (int)segs.size();
    jpeg_segments(data + b, len, P, segs, b, k);
    P.img.nseg = (int)segs.size() - P.img.seg0;
    imgs[k] = P.img;
  }
  jpeg_long_segments(data, segs, longs);
  if (!longs.empty() && (int64_t)longs.back().sub0 + longs.back().nsub > INT32_MAX / 2) {
    set_error("udh_jpeg_plan: too much entropy-coded data for one plan");
    return UDH_EINVAL;
  }
  return UDH_OK;
}

// header | images | segments | long segments (none: the plan is laid out as it was before the parallel path existed)
static_assert(sizeof(JpegSeg) % 16 == 0 && sizeof(JpegLong) % 16 == 0, "plan sections must stay 16-byte aligned");
static size_t plan_longs_offset(int n, size_t nseg) {
  return align_up(sizeof(JpegPlanHeader), 16) + align_up((size_t)n * sizeof(JpegImage), 16) + nseg * sizeof(JpegSeg);
}
static size_t plan_size(int n, size_t nseg, size_t nlong) { return plan_longs_offset(n, nseg) + nlong * sizeof(JpegLong); }

// Parallel-path workspace after the coefficient and sample planes: per subsequence two JpegSubRes (ping-pong rounds), a
// JpegPState and a JpegSubOut; per long segment kJpegMaxRounds + 1 change flags; per segment one done byte.
struct JpegParWs {
  size_t res, used, outp, changed, done, end;
};
static JpegParWs jpeg_par_ws(size_t base, int64_t nsub, int nlong, int nseg) {
  JpegParWs o;
  o.res = align_up(base, 16);
  o.used = o.res + align_up(2 * (size_t)nsub * sizeof(JpegSubRes), 16);
  o.outp = o.used + align_up((size_t)nsub * sizeof(JpegPState), 16);
  o.changed = o.outp + align_up((size_t)nsub * sizeof(JpegSubOut), 16);
  o.done = o.changed + align_up((size_t)nlong * (kJpegMaxRounds + 1) * sizeof(int32_t), 16);
  o.end = o.done + align_up((size_t)nseg, 16);
  return o;
}

}  // namespace udh

using namespace udh;

static int g_jpeg_lanes = 32;
static int g_jpeg_rounds = kJpegMaxRounds;

extern "C" int udh_jpeg_parse(const uint8_t* data, int64_t nbytes, udh_jpeg_info* info) {
  UDH_REQUIRE(info && (data || nbytes == 0) && nbytes >= 0, "udh_jpeg_parse: bad argument");
  JpegParsed P;
  const int r = jpeg_parse_impl(data, nbytes, P);
  *info = P.info;
  info->reason = r;
  return UDH_OK;
}

extern "C" size_t udh_jpeg_plan_bytes(const uint8_t* data, const int64_t* offsets, int n, int h, int w) {
  if (!data || !offsets || n < 1 || h < 1 || w < 1) return 0;
  std::vector<JpegImage> imgs;
  std::vector<JpegSeg> segs;
  std::vector<JpegLong> longs;
  if (jpeg_build_plan(data, offsets, n, h, w, imgs, segs, longs) != UDH_OK) return 0;
  return plan_size(n, segs.size(), longs.size());
}

extern "C" int udh_jpeg_plan(const uint8_t* data, const int64_t* offsets, int n, int h, int w, void* plan, size_t plan_bytes) {
  UDH_REQUIRE(data && offsets && plan, "udh_jpeg_plan: null pointer");
  UDH_REQUIRE(n >= 1 && h >= 1 && w >= 1 && h <= 65535 && w <= 65535, "udh_jpeg_plan: bad dimensions");
  std::vector<JpegImage> imgs;
  std::vector<JpegSeg> segs;
  std::vector<JpegLong> longs;
  const int rc = jpeg_build_plan(data, offsets, n, h, w, imgs, segs, longs);
  if (rc != UDH_OK) return rc;
  const size_t need = plan_size(n, segs.size(), longs.size());
  if (plan_bytes < need) {
    set_error("udh_jpeg_plan: plan buffer of %zu bytes, %zu needed", plan_bytes, need);
    return UDH_EWS;
  }
  uint8_t* p = static_cast<uint8_t*>(plan);
  JpegPlanHeader hd{};
  hd.magic = kJpegMagic;
  hd.n = n; hd.h = h; hd.w = w; hd.nseg = (int)segs.size(); hd.nlong = (int)longs.size();
  hd.bytes = (int64_t)need;
  hd.plane = jpeg_plane_coefs(h, w);
  memcpy(p, &hd, sizeof(hd));
  p += align_up(sizeof(JpegPlanHeader), 16);
  memcpy(p, imgs.data(), (size_t)n * sizeof(JpegImage));
  p += align_up((size_t)n * sizeof(JpegImage), 16);
  memcpy(p, segs.data(), segs.size() * sizeof(JpegSeg));
  p += segs.size() * sizeof(JpegSeg);
  if (!longs.empty()) memcpy(p, longs.data(), longs.size() * sizeof(JpegLong));
  return UDH_OK;
}

extern "C" size_t udh_jpeg_workspace_bytes(int n, int h, int w) {
  if (n < 1 || h < 1 || w < 1) return 0;
  return (size_t)n * 3 * (size_t)jpeg_plane_coefs(h, w) * (sizeof(int16_t) + sizeof(uint8_t));
}

// the plan's long segments and their subsequence count (host copy of the plan)
static const JpegLong* plan_longs(const JpegPlanHeader& hd, const void* plan, int64_t* nsub, int* max_nsub) {
  const JpegLong* L = reinterpret_cast<const JpegLong*>(static_cast<const uint8_t*>(plan) + plan_longs_offset(hd.n, hd.nseg));
  *nsub = hd.nlong ? (int64_t)L[hd.nlong - 1].sub0 + L[hd.nlong - 1].nsub : 0;
  *max_nsub = 0;
  for (int k = 0; k < hd.nlong; ++k) *max_nsub = std::max(*max_nsub, L[k].nsub);
  return L;
}

extern "C" size_t udh_jpeg_plan_workspace_bytes(const void* plan_host) {
  if (!plan_host) return 0;
  JpegPlanHeader hd;
  memcpy(&hd, plan_host, sizeof(hd));
  if (hd.magic != kJpegMagic || hd.n < 1) return 0;
  const size_t base = udh_jpeg_workspace_bytes(hd.n, hd.h, hd.w);
  if (hd.nlong == 0) return base;
  int64_t nsub;
  int max_nsub;
  plan_longs(hd, plan_host, &nsub, &max_nsub);
  return jpeg_par_ws(base, nsub, hd.nlong, hd.nseg).end;
}

extern "C" int udh_jpeg_decode(const void* plan_host, const void* plan_dev, const uint8_t* data, uint8_t* out, int32_t* status,
                               void* ws, size_t ws_bytes, void* stream) {
  UDH_REQUIRE(plan_host && plan_dev && data && out && status && ws, "udh_jpeg_decode: null pointer");
  JpegPlanHeader hd;
  memcpy(&hd, plan_host, sizeof(hd));
  UDH_REQUIRE(hd.magic == kJpegMagic && hd.n >= 1, "udh_jpeg_decode: not a plan made by udh_jpeg_plan");
  const size_t need = udh_jpeg_plan_workspace_bytes(plan_host);
  if (ws_bytes < need) {
    set_error("udh_jpeg_decode: workspace of %zu bytes, %zu needed", ws_bytes, need);
    return UDH_EWS;
  }
  UDH_REQUIRE(((uintptr_t)ws & 15) == 0 && ((uintptr_t)plan_dev & 15) == 0, "udh_jpeg_decode: plan and workspace must be 16-byte aligned");
  cudaStream_t st = as_stream(stream);
  const uint8_t* pd = static_cast<const uint8_t*>(plan_dev);
  const JpegImage* imgs = reinterpret_cast<const JpegImage*>(pd + align_up(sizeof(JpegPlanHeader), 16));
  const JpegSeg* segs = reinterpret_cast<const JpegSeg*>(pd + align_up(sizeof(JpegPlanHeader), 16) + align_up((size_t)hd.n * sizeof(JpegImage), 16));
  int16_t* coef = static_cast<int16_t*>(ws);
  uint8_t* samples = reinterpret_cast<uint8_t*>(coef + (size_t)hd.n * 3 * hd.plane);
  UDH_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t) * hd.n, st));
  int rc;
  uint8_t* done = nullptr;
  JpegSubRes* res = nullptr;
  JpegPState* used = nullptr;
  JpegSubOut* outp = nullptr;
  const JpegLong* longs_d = nullptr;
  int64_t nsub = 0;
  int max_nsub = 0;
  if (hd.nlong) {   // parallel path: rounds, scan (segments that synchronised are marked done for the serial kernel)
    plan_longs(hd, plan_host, &nsub, &max_nsub);
    const JpegParWs o = jpeg_par_ws(udh_jpeg_workspace_bytes(hd.n, hd.h, hd.w), nsub, hd.nlong, hd.nseg);
    uint8_t* w8 = static_cast<uint8_t*>(ws);
    res = reinterpret_cast<JpegSubRes*>(w8 + o.res);
    used = reinterpret_cast<JpegPState*>(w8 + o.used);
    outp = reinterpret_cast<JpegSubOut*>(w8 + o.outp);
    int32_t* changed = reinterpret_cast<int32_t*>(w8 + o.changed);
    done = w8 + o.done;
    longs_d = reinterpret_cast<const JpegLong*>(pd + plan_longs_offset(hd.n, hd.nseg));
    UDH_CUDA(cudaMemsetAsync(w8 + o.changed, 0, o.end - o.changed, st));
    const dim3 grid((max_nsub + 127) / 128, hd.nlong);
    for (int r = 0; r <= g_jpeg_rounds; ++r) {
      jpeg_sync_kernel<<<grid, 128, 0, st>>>(imgs, segs, longs_d, data, res, used, changed, nsub, r);
      if ((rc = check_launch("jpeg_sync"))) return rc;
    }
    jpeg_scan_kernel<<<hd.nlong, 1024, 0, st>>>(imgs, segs, longs_d, res, changed, outp, done, status, nsub, g_jpeg_rounds);
    if ((rc = check_launch("jpeg_scan"))) return rc;
  }
  const int ctas = (hd.n + kJpegImgsPerCta - 1) / kJpegImgsPerCta;
  if (g_jpeg_lanes == 1)
    jpeg_entropy_kernel<1><<<ctas, kJpegImgsPerCta * 1, 0, st>>>(imgs, segs, data, coef, hd.plane, status, hd.n, done);
  else
    jpeg_entropy_kernel<32><<<ctas, kJpegImgsPerCta * 32, 0, st>>>(imgs, segs, data, coef, hd.plane, status, hd.n, done);
  if ((rc = check_launch("jpeg_entropy"))) return rc;
  if (hd.nlong) {
    jpeg_write_kernel<<<dim3((max_nsub + 127) / 128, hd.nlong), 128, 0, st>>>(imgs, segs, longs_d, data, used, outp, done, coef,
                                                                               hd.plane);
    if ((rc = check_launch("jpeg_write"))) return rc;
  }
  const int maxblk = (int)(3 * hd.plane / 64);
  jpeg_idct_kernel<<<dim3((maxblk + 127) / 128, hd.n), 128, 0, st>>>(imgs, coef, samples, hd.plane);
  rc = check_launch("jpeg_idct");
  if (rc) return rc;
  const int npx = hd.h * hd.w;
  jpeg_color_kernel<<<dim3(min((npx + 255) / 256, 64), hd.n), 256, 0, st>>>(imgs, samples, hd.plane, out, hd.h, hd.w);
  return check_launch("udh_jpeg_decode");
}

extern "C" int udh_debug_jpeg_set_parallel(int mode) {
  UDH_REQUIRE(mode >= -1 && mode <= 1, "udh_debug_jpeg_set_parallel: mode must be -1 (by segment length), 0 (off) or 1 (on)");
  g_jpeg_parallel = mode;
  return UDH_OK;
}

extern "C" int udh_debug_jpeg_set_sync_rounds(int rounds) {
  UDH_REQUIRE(rounds >= 0 && rounds <= kJpegMaxRounds, "udh_debug_jpeg_set_sync_rounds: rounds must be 0..16");
  g_jpeg_rounds = rounds;
  return UDH_OK;
}

extern "C" int udh_debug_jpeg_parallel_segments(const void* plan_host, const void* ws, int32_t* count) {
  UDH_REQUIRE(plan_host && ws && count, "udh_debug_jpeg_parallel_segments: null pointer");
  JpegPlanHeader hd;
  memcpy(&hd, plan_host, sizeof(hd));
  UDH_REQUIRE(hd.magic == kJpegMagic && hd.n >= 1, "udh_debug_jpeg_parallel_segments: not a plan made by udh_jpeg_plan");
  *count = 0;
  if (!hd.nlong) return UDH_OK;
  int64_t nsub;
  int max_nsub;
  plan_longs(hd, plan_host, &nsub, &max_nsub);
  const JpegParWs o = jpeg_par_ws(udh_jpeg_workspace_bytes(hd.n, hd.h, hd.w), nsub, hd.nlong, hd.nseg);
  std::vector<uint8_t> done(hd.nseg);
  UDH_CUDA(cudaMemcpy(done.data(), static_cast<const uint8_t*>(ws) + o.done, hd.nseg, cudaMemcpyDeviceToHost));
  for (uint8_t d : done) *count += d;
  return UDH_OK;
}

extern "C" int udh_debug_jpeg_set_lanes(int lanes) {
  UDH_REQUIRE(lanes == 1 || lanes == 32, "udh_debug_jpeg_set_lanes: lanes must be 1 or 32");
  g_jpeg_lanes = lanes;
  return UDH_OK;
}
