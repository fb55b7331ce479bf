// Graph-cut seams: cv2.detail's GraphCutSeamFinder(COST_COLOR) as the canonical minimum cut (the rule: oracle/seam_gc.py),
// on the seam pool and frame table of udh_mosaic_seam_gc_masks_u8 (warp_perspective.cu), and the grid min-cut it runs
// (udh_debug_grid_mincut).
#include <algorithm>
#include <climits>
#include <cstdint>
#include <vector>

#include "roi_warp.cuh"

namespace udh {

// ---- graph-cut seams: cv2.detail's GraphCutSeamFinder (COST_COLOR) as the canonical minimum cut (oracle/seam_gc.py) -----
// A pair's window (the Voronoi finder's) is a 4-connected grid graph with integer capacities: edge (p, q) carries
// d(p) + d(q) + 1 (+ GC_PENALTY unless both masks hold p and q) both ways, d the squared RGB difference of the two ROI
// warps; a pixel held by frame i alone is tied to the source, one held by frame j alone to the sink, with GC_TERM.  Every
// capacity is below 2^24 and every excess below 2^31, so the flow runs in int32.  T, the pixels that reach the sink in the
// residual graph of a maximum preflow, is the same for every maximum preflow: the racy parallel flow below leaves
// deterministic bytes.
// The flow is synchronous push-relabel.  A push phase moves excess along admissible edges only (h(p) = h(q) + 1), so no
// edge is pushed from both ends in one phase and only the excess needs atomics; a relabel phase lifts every active pixel
// to 1 + its lowest residual neighbour (heights only grow, so a racy read still gives a valid labelling).  Every few
// phases a global relabel recomputes the exact distance to the sink by tile-wise BFS relaxation (GC_INF: the pixel cannot
// reach it, so its excess is stranded for good); the flow is maximum when no pixel holding excess has a finite height,
// and those heights are then T's complement.
constexpr int GC_TERM = 10000, GC_PENALTY = 1000, GC_CAP_MAX = 1 << 24, GC_INF = INT_MAX;
constexpr int GC_TILE = 32, GC_BFS_BATCH = 4;   // BFS tiles of 32 x 32 pixels (32 x 8 threads, 4 rows each)

struct GcGrid {
  int w, h;
  int64_t n;
  int* r[4];            // residual capacity to the right, lower, left and upper neighbour (0 across the border)
  int* e;               // excess
  int* t;               // residual capacity to the sink
  int* ht;              // height: a lower bound of the residual distance to the sink, GC_INF when there is none
  int* src;             // the source and sink capacities as given
  int* snk;
};

__device__ __forceinline__ int64_t gc_nbr(const GcGrid& g, int64_t p, int d) {
  return d == 0 ? p + 1 : d == 1 ? p + g.w : d == 2 ? p - 1 : p - g.w;
}

__device__ __forceinline__ int gc_ld(const int* p) { return *reinterpret_cast<const volatile int*>(p); }

// Debug grid: right / down capacity planes (the last column's / row's ignored) and the terminals, checked against
// [0, GC_CAP_MAX] (bad[0] set otherwise).
__global__ void __launch_bounds__(256) gc_grid_init_kernel(GcGrid g, const int* __restrict__ hcap, const int* __restrict__ vcap,
                                                           const int* __restrict__ src, const int* __restrict__ snk, int* bad) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < g.n; p += (int64_t)gridDim.x * blockDim.x) {
    const int y = (int)(p / g.w), x = (int)(p - (int64_t)y * g.w);
    const int c[4] = {x + 1 < g.w ? hcap[p] : 0, y + 1 < g.h ? vcap[p] : 0, x > 0 ? hcap[p - 1] : 0, y > 0 ? vcap[p - g.w] : 0};
    const int s = src[p], k = snk[p];
    bool ok = s >= 0 && s <= GC_CAP_MAX && k >= 0 && k <= GC_CAP_MAX;
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      ok = ok && c[d] >= 0 && c[d] <= GC_CAP_MAX;
      g.r[d][p] = c[d];
    }
    if (!ok) atomicOr(bad, 1);
    g.e[p] = g.src[p] = s;
    g.t[p] = g.snk[p] = k;
  }
}

// Seam window, first pass: per window pixel, d(p) (the warps are 0 outside their ROIs) | s_i << 20 | s_j << 21 into ht.
__global__ void __launch_bounds__(256) gc_window_color_kernel(GcGrid g, const SeamFrame* __restrict__ fr, const double* __restrict__ M,
                                                            const uint8_t* __restrict__ seam, int fi, int fj, int wx0, int wy0) {
  __shared__ double mi[2][9];
  if (threadIdx.x < 2) cv_invert3(M + (int64_t)(threadIdx.x ? fj : fi) * 9, mi[threadIdx.x]);
  __syncthreads();
  const SeamFrame* F[2] = {fr + fi, fr + fj};
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < g.n; p += (int64_t)gridDim.x * blockDim.x) {
    const int y = (int)(p / g.w), x = (int)(p - (int64_t)y * g.w);
    int v[2][3], s[2];
#pragma unroll
    for (int f = 0; f < 2; ++f) {
      const SeamFrame* Fk = F[f];
      const SeamRect r{__ldg(&Fk->off), __ldg(&Fk->rx), __ldg(&Fk->ry), __ldg(&Fk->rw), __ldg(&Fk->rh)};
      const int lx = wx0 + x - r.rx, ly = wy0 + y - r.ry;
      s[f] = seam_at(seam, r, wx0 + x, wy0 + y);
      v[f][0] = v[f][1] = v[f][2] = 0;
      if ((unsigned)lx < (unsigned)r.rw && (unsigned)ly < (unsigned)r.rh) {
        const uint8_t* src = reinterpret_cast<const uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&Fk->src)));
        mb_roi_warp(src, __ldg(&Fk->h), __ldg(&Fk->w), mi[f], lx, ly, __ldg(&Fk->bw), v[f]);
      }
    }
    int d = 0;
#pragma unroll
    for (int c = 0; c < 3; ++c) d += (v[0][c] - v[1][c]) * (v[0][c] - v[1][c]);
    g.ht[p] = d | s[0] << 20 | s[1] << 21;
  }
}

// Seam window, second pass: the capacities and terminals from the first pass's words.
__global__ void __launch_bounds__(256) gc_window_graph_kernel(GcGrid g) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < g.n; p += (int64_t)gridDim.x * blockDim.x) {
    const int y = (int)(p / g.w), x = (int)(p - (int64_t)y * g.w);
    const int a = g.ht[p];
    const bool in[4] = {x + 1 < g.w, y + 1 < g.h, x > 0, y > 0};
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      int c = 0;
      if (in[d]) {
        const int b = g.ht[gc_nbr(g, p, d)];
        c = (a & 0xfffff) + (b & 0xfffff) + 1 + ((a & b) >> 20 == 3 ? 0 : GC_PENALTY);
      }
      g.r[d][p] = c;
    }
    const int si = a >> 20 & 1, sj = a >> 21 & 1;
    g.e[p] = g.src[p] = si && !sj ? GC_TERM : 0;
    g.t[p] = g.snk[p] = sj && !si ? GC_TERM : 0;
  }
}

// Push phase: every active pixel sends its excess to the sink, then along its admissible edges.  Only p writes r[.][p]
// and the reverse residuals of the edges it pushes along (an admissible edge is never admissible the other way).
__global__ void __launch_bounds__(256) gc_push_kernel(GcGrid g) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < g.n; p += (int64_t)gridDim.x * blockDim.x) {
    const int ex = gc_ld(g.e + p), hp = g.ht[p];
    if (ex <= 0 || hp == GC_INF) continue;
    int sent = 0;
    const int tp = g.t[p];
    if (tp > 0) {
      sent = min(ex, tp);
      g.t[p] = tp - sent;
    }
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      const int rc = g.r[d][p];
      if (sent == ex || rc <= 0) continue;
      const int64_t q = gc_nbr(g, p, d);
      if (g.ht[q] != hp - 1) continue;
      const int f = min(ex - sent, rc);
      g.r[d][p] = rc - f;
      g.r[d ^ 2][q] += f;
      atomicAdd(g.e + q, f);
      sent += f;
    }
    if (sent) atomicSub(g.e + p, sent);
  }
}

// Relabel phase: every active pixel to 1 + its lowest residual neighbour (1 with a residual sink edge), GC_INF when that
// exceeds the pixel count (no residual path is that long).
__global__ void __launch_bounds__(256) gc_relabel_kernel(GcGrid g) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < g.n; p += (int64_t)gridDim.x * blockDim.x) {
    const int hp = g.ht[p];
    if (g.e[p] <= 0 || hp == GC_INF) continue;
    int m = g.t[p] > 0 ? 1 : GC_INF;
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      if (g.r[d][p] <= 0) continue;
      const int hq = gc_ld(g.ht + gc_nbr(g, p, d));
      if (hq != GC_INF) m = min(m, hq + 1);
    }
    if (m != GC_INF && m > g.n) m = GC_INF;
    if (m > hp) g.ht[p] = m;
  }
}

__global__ void __launch_bounds__(256) gc_bfs_init_kernel(GcGrid g) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < g.n; p += (int64_t)gridDim.x * blockDim.x)
    g.ht[p] = g.t[p] > 0 ? 1 : GC_INF;
}

// One pass of the global relabel: each CTA relaxes its tile's heights in shared memory, h(p) = min(h(p), 1 + h(q)) over
// residual edges p -> q (the halo read once from global memory), until the tile stops changing, then stores them.
// flags[0] is set when any height changed, flags[1] when a pixel holding excess has a finite height.  Heights only fall
// and always bound a real path, so the passes may read each other's stores in any order.
__global__ void __launch_bounds__(GC_TILE * 8) gc_bfs_kernel(GcGrid g, int* flags) {
  __shared__ int sh[GC_TILE + 2][GC_TILE + 2];
  const int tx = threadIdx.x & (GC_TILE - 1), ty = threadIdx.x / GC_TILE;
  const int x0 = blockIdx.x * GC_TILE, y0 = blockIdx.y * GC_TILE;
  for (int i = threadIdx.x; i < (GC_TILE + 2) * (GC_TILE + 2); i += blockDim.x) {
    const int ly = i / (GC_TILE + 2), lx = i - ly * (GC_TILE + 2), gx = x0 + lx - 1, gy = y0 + ly - 1;
    sh[ly][lx] = gx >= 0 && gx < g.w && gy >= 0 && gy < g.h ? gc_ld(g.ht + (int64_t)gy * g.w + gx) : GC_INF;
  }
  int res[4], h0[4];
  const int x = x0 + tx;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int y = y0 + ty + 8 * k;
    res[k] = 0;
    if (x < g.w && y < g.h) {
      const int64_t p = (int64_t)y * g.w + x;
#pragma unroll
      for (int d = 0; d < 4; ++d) res[k] |= (g.r[d][p] > 0) << d;
      res[k] |= 16;                                                   // an in-grid pixel
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) h0[k] = sh[ty + 8 * k + 1][tx + 1];
  for (int it = 0; it < GC_TILE * GC_TILE; ++it) {
    bool ch = false;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (!res[k]) continue;
      const int ly = ty + 8 * k + 1, lx = tx + 1, cur = sh[ly][lx];
      int m = cur;
      if (res[k] & 1) m = min(m, sh[ly][lx + 1]);
      if (res[k] & 2) m = min(m, sh[ly + 1][lx]);
      if (res[k] & 4) m = min(m, sh[ly][lx - 1]);
      if (res[k] & 8) m = min(m, sh[ly - 1][lx]);
      if (m != GC_INF && m + 1 < cur) {
        sh[ly][lx] = m + 1;
        ch = true;
      }
    }
    if (!__syncthreads_or(ch)) break;
  }
  bool changed = false, active = false;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (!res[k]) continue;
    const int y = y0 + ty + 8 * k, hv = sh[ty + 8 * k + 1][tx + 1];
    const int64_t p = (int64_t)y * g.w + x;
    if (hv != h0[k]) {
      g.ht[p] = hv;
      changed = true;
    }
    if (hv != GC_INF && g.e[p] > 0) active = true;
  }
  changed = __syncthreads_or(changed);
  active = __syncthreads_or(active);
  if (threadIdx.x == 0) {
    if (changed) atomicOr(flags, 1);
    if (active) atomicOr(flags + 1, 1);
  }
}

// The cut: S = {ht = GC_INF}.  Adds its capacity (sink edges of S, source edges of T, and edges S -> T, each edge's
// capacity half the sum of its two residuals) to *cut; writes T (1 / 0) to tout if given; and, given a seam pool, updates
// the pair's masks over the intersection (window pixels [gap, gap + iw) x [gap, gap + ih)): where p is in S and frame a
// holds it frame b's mask is cleared, where p is in T and frame b holds it frame a's.
__global__ void __launch_bounds__(256) gc_cut_kernel(GcGrid g, unsigned long long* cut, uint8_t* __restrict__ tout,
                                                     uint8_t* __restrict__ seam, SeamRect a, SeamRect b, int wx0, int wy0, int gap,
                                                     int iw, int ih) {
  long long sum = 0;
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < g.n; p += (int64_t)gridDim.x * blockDim.x) {
    const int y = (int)(p / g.w), x = (int)(p - (int64_t)y * g.w);
    const bool inS = g.ht[p] == GC_INF;
    if (inS) {
      sum += g.snk[p];
#pragma unroll
      for (int d = 0; d < 4; ++d) {
        const int rp = g.r[d][p];
        const int64_t q = gc_nbr(g, p, d);
        const bool in = d == 0 ? x + 1 < g.w : d == 1 ? y + 1 < g.h : d == 2 ? x > 0 : y > 0;
        if (in && g.ht[q] != GC_INF) sum += ((long long)rp + g.r[d ^ 2][q]) / 2;
      }
    } else {
      sum += g.src[p];
    }
    if (tout) tout[p] = inS ? 0 : 1;
    if (seam && x >= gap && x < gap + iw && y >= gap && y < gap + ih) {
      const int cx = wx0 + x, cy = wy0 + y;
      if (inS) {
        if (seam_at(seam, a, cx, cy)) seam[b.off + (int64_t)(cy - b.ry) * b.rw + (cx - b.rx)] = 0;
      } else {
        if (seam_at(seam, b, cx, cy)) seam[a.off + (int64_t)(cy - a.ry) * a.rw + (cx - a.rx)] = 0;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_down_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0 && sum) atomicAdd(cut, (unsigned long long)sum);
}

static size_t gc_align(size_t v) { return (v + 255) & ~(size_t)255; }

static unsigned gc_blocks(int64_t px) {
  const int64_t b = (px + 255) / 256;
  return (unsigned)(b < 1 ? 1 : b > 4096 ? 4096 : b);
}

// A grid graph's planes in a workspace, after its first off bytes: nine int32 planes of n pixels (r[4], e, t, ht, src,
// snk), the BFS passes' flags and the bad-input flag, then ncut uint64 cut values.
struct GcLayout {
  int64_t n;
  size_t planes, flags, cuts, total;
};

static GcLayout gc_layout(size_t off, int64_t n, int64_t ncut) {
  GcLayout L;
  L.n = n;
  L.planes = gc_align(off);
  L.flags = gc_align(L.planes + 9 * (size_t)n * sizeof(int));
  L.cuts = gc_align(L.flags + (2 * GC_BFS_BATCH + 1) * sizeof(int));
  L.total = gc_align(L.cuts + (size_t)ncut * sizeof(unsigned long long));
  return L;
}

static GcGrid gc_grid(char* base, const GcLayout& L, int w, int h) {
  GcGrid g;
  g.w = w;
  g.h = h;
  g.n = (int64_t)w * h;
  int* pl = reinterpret_cast<int*>(base + L.planes);
  for (int d = 0; d < 4; ++d) g.r[d] = pl + d * L.n;
  g.e = pl + 4 * L.n;
  g.t = pl + 5 * L.n;
  g.ht = pl + 6 * L.n;
  g.src = pl + 7 * L.n;
  g.snk = pl + 8 * L.n;
  return g;
}

// Global relabel: exact residual distances to the sink in g.ht; active: a pixel holding excess reaches the sink.  Passes
// go out GC_BFS_BATCH at a time and stop at the first that changes nothing (each pass that changes something settles at
// least one more pixel, so at most n + 1 of them).
static int gc_bfs(const GcGrid& g, int* flags, cudaStream_t st, bool& active, const char* what) {
  gc_bfs_init_kernel<<<gc_blocks(g.n), 256, 0, st>>>(g);
  int rc = check_launch(what);
  if (rc != UDH_OK) return rc;
  const dim3 grid((unsigned)((g.w + GC_TILE - 1) / GC_TILE), (unsigned)((g.h + GC_TILE - 1) / GC_TILE));
  int host[2 * GC_BFS_BATCH];
  for (int64_t pass = 0; pass <= g.n + GC_BFS_BATCH; pass += GC_BFS_BATCH) {
    UDH_CUDA(cudaMemsetAsync(flags, 0, sizeof(host), st));
    for (int k = 0; k < GC_BFS_BATCH; ++k) {
      gc_bfs_kernel<<<grid, GC_TILE * 8, 0, st>>>(g, flags + 2 * k);
      if ((rc = check_launch(what)) != UDH_OK) return rc;
    }
    UDH_CUDA(cudaMemcpyAsync(host, flags, sizeof(host), cudaMemcpyDeviceToHost, st));
    UDH_CUDA(cudaStreamSynchronize(st));
    for (int k = 0; k < GC_BFS_BATCH; ++k)
      if (!host[2 * k]) {
        active = host[2 * k + 1] != 0;
        return UDH_OK;
      }
  }
  set_error("%s: the global relabel of a %dx%d grid did not settle within %lld passes", what, g.h, g.w, (long long)(g.n + 1));
  return UDH_ECUDA;
}

// A maximum preflow of g (initialised: capacities, e = src, t = snk), its sink side left as the finite heights of g.ht.
// Push-relabel phases go out between global relabels, 64 at first, doubling up to twice the grid's perimeter.  The phases
// are capped at 4 n + 4096 in all, and the call fails past the cap rather than spin.  The cap is a heuristic, not a
// worst-case bound (push-relabel may need O(n^2) phases): the windows of a 1080 x 1920 and a 12 MP sweep settle within
// 1 % of it, since a global relabel strands every excess that can no longer reach the sink.
static int gc_maxflow(const GcGrid& g, int* flags, cudaStream_t st, const char* what) {
  const int64_t bound = 4 * g.n + 4096, most = 4 * ((int64_t)g.w + g.h) + 64;
  int64_t phases = 0, K = 64;
  for (;;) {
    bool active = false;
    int rc = gc_bfs(g, flags, st, active, what);
    if (rc != UDH_OK) return rc;
    if (!active) return UDH_OK;
    if (phases >= bound) {
      set_error("%s: the flow of a %dx%d grid did not settle within %lld push-relabel phases", what, g.h, g.w, (long long)bound);
      return UDH_ECUDA;
    }
    K = std::min(K, bound - phases);                                // the last round stops at the cap
    for (int64_t k = 0; k < K; ++k) {
      gc_push_kernel<<<gc_blocks(g.n), 256, 0, st>>>(g);
      if ((rc = check_launch(what)) != UDH_OK) return rc;
      gc_relabel_kernel<<<gc_blocks(g.n), 256, 0, st>>>(g);
      if ((rc = check_launch(what)) != UDH_OK) return rc;
    }
    phases += K;
    K = std::min(2 * K, most);
  }
}

size_t gc_workspace_bytes(size_t off, int64_t max_win, int64_t npairs) { return gc_layout(off, max_win, npairs).total; }

int gc_seam_pairs(char* base, size_t off, int64_t max_win, const SeamFrame* fr, const std::vector<SeamFrame>& host, const double* M,
                  uint8_t* seam, const std::vector<int>& pi, const std::vector<int>& pj, int64_t* cut, cudaStream_t st, const char* what) {
  const size_t npairs = pi.size();
  const GcLayout L = gc_layout(off, max_win, (int64_t)npairs);
  int* flags = reinterpret_cast<int*>(base + L.flags);
  unsigned long long* cuts = reinterpret_cast<unsigned long long*>(base + L.cuts);
  if (npairs) UDH_CUDA(cudaMemsetAsync(cuts, 0, npairs * sizeof(unsigned long long), st));
  int rc;
  for (size_t q = 0; q < npairs; ++q) {
    const SeamFrame &A = host[pi[q]], &B = host[pj[q]];
    const SeamRect a{A.off, A.rx, A.ry, A.rw, A.rh}, b{B.off, B.rx, B.ry, B.rw, B.rh};
    const int x0 = std::max(A.rx, B.rx), y0 = std::max(A.ry, B.ry);
    const int iw = std::min(A.rx + A.rw, B.rx + B.rw) - x0, ih = std::min(A.ry + A.rh, B.ry + B.rh) - y0;
    const GcGrid g = gc_grid(base, L, iw + 2 * SEAM_GAP, ih + 2 * SEAM_GAP);
    const int wx0 = x0 - SEAM_GAP, wy0 = y0 - SEAM_GAP;
    gc_window_color_kernel<<<gc_blocks(g.n), 256, 0, st>>>(g, fr, M, seam, pi[q], pj[q], wx0, wy0);
    if ((rc = check_launch("udh_mosaic_seam_gc_masks_u8 (color)")) != UDH_OK) return rc;
    gc_window_graph_kernel<<<gc_blocks(g.n), 256, 0, st>>>(g);
    if ((rc = check_launch("udh_mosaic_seam_gc_masks_u8 (graph)")) != UDH_OK) return rc;
    if ((rc = gc_maxflow(g, flags, st, what)) != UDH_OK) return rc;
    gc_cut_kernel<<<gc_blocks(g.n), 256, 0, st>>>(g, cuts + q, nullptr, seam, a, b, wx0, wy0, SEAM_GAP, iw, ih);
    if ((rc = check_launch("udh_mosaic_seam_gc_masks_u8 (cut)")) != UDH_OK) return rc;
  }
  if (cut && npairs) {
    std::vector<unsigned long long> c(npairs);
    UDH_CUDA(cudaMemcpyAsync(c.data(), cuts, npairs * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    UDH_CUDA(cudaStreamSynchronize(st));
    for (size_t q = 0; q < npairs; ++q) cut[q] = (int64_t)c[q];
  }
  return UDH_OK;
}

}  // namespace udh

using namespace udh;

constexpr int GC_MAX_SIDE = 32766 + 2 * SEAM_GAP;   // a seam window's largest side

extern "C" size_t udh_debug_grid_mincut_workspace_bytes(int h, int w) {
  return h >= 1 && w >= 1 && h <= GC_MAX_SIDE && w <= GC_MAX_SIDE ? gc_layout(0, (int64_t)h * w, 1).total : 0;
}

extern "C" int udh_debug_grid_mincut(const int32_t* hcap, const int32_t* vcap, const int32_t* src, const int32_t* snk, int h, int w,
                                     uint8_t* T, int64_t* cut, int32_t* residual, void* ws, size_t ws_bytes, void* stream) {
  const char* what = "udh_debug_grid_mincut";
  UDH_REQUIRE(hcap && vcap && src && snk && T && cut && ws, "%s: null pointer", what);
  UDH_REQUIRE(h >= 1 && w >= 1 && h <= GC_MAX_SIDE && w <= GC_MAX_SIDE, "%s: bad dimensions %dx%d (sides 1..%d)", what, h, w, GC_MAX_SIDE);
  const GcLayout L = gc_layout(0, (int64_t)h * w, 1);
  if (ws_bytes < L.total) {
    set_error("%s: workspace of %zu bytes, %zu needed", what, ws_bytes, L.total);
    return UDH_EWS;
  }
  const cudaStream_t st = as_stream(stream);
  char* base = static_cast<char*>(ws);
  int* flags = reinterpret_cast<int*>(base + L.flags);
  unsigned long long* cuts = reinterpret_cast<unsigned long long*>(base + L.cuts);
  const GcGrid g = gc_grid(base, L, w, h);
  UDH_CUDA(cudaMemsetAsync(flags + 2 * GC_BFS_BATCH, 0, sizeof(int), st));
  UDH_CUDA(cudaMemsetAsync(cuts, 0, sizeof(unsigned long long), st));
  gc_grid_init_kernel<<<gc_blocks(g.n), 256, 0, st>>>(g, hcap, vcap, src, snk, flags + 2 * GC_BFS_BATCH);
  int rc = check_launch("udh_debug_grid_mincut (init)");
  if (rc != UDH_OK) return rc;
  int bad = 0;
  UDH_CUDA(cudaMemcpyAsync(&bad, flags + 2 * GC_BFS_BATCH, sizeof(int), cudaMemcpyDeviceToHost, st));
  UDH_CUDA(cudaStreamSynchronize(st));
  UDH_REQUIRE(!bad, "%s: a capacity lies outside [0, %d]", what, GC_CAP_MAX);
  if ((rc = gc_maxflow(g, flags, st, what)) != UDH_OK) return rc;
  gc_cut_kernel<<<gc_blocks(g.n), 256, 0, st>>>(g, cuts, T, nullptr, SeamRect{}, SeamRect{}, 0, 0, 0, 0, 0);
  if ((rc = check_launch("udh_debug_grid_mincut (cut)")) != UDH_OK) return rc;
  if (residual) {
    UDH_CUDA(cudaMemcpyAsync(residual, g.r[0], 4 * (size_t)g.n * sizeof(int), cudaMemcpyDeviceToDevice, st));
    UDH_CUDA(cudaMemcpyAsync(residual + 4 * g.n, g.t, (size_t)g.n * sizeof(int), cudaMemcpyDeviceToDevice, st));
  }
  unsigned long long c = 0;
  UDH_CUDA(cudaMemcpyAsync(&c, cuts, sizeof(c), cudaMemcpyDeviceToHost, st));
  UDH_CUDA(cudaStreamSynchronize(st));
  *cut = (int64_t)c;
  return UDH_OK;
}
