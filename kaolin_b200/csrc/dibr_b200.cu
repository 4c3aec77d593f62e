// dibr_b200.cu — hand-written sm_90a kernels + C ABI (include/dibr_b200.h) for
// Kaolin's DIB-R hot path.  See DESIGN.md for the data layout and the roofline
// of each kernel.  Reference behaviour being reproduced:
//   kaolin/csrc/render/mesh/rasterization_cuda.cu   (forward :43-192, backward :238-402)
//   kaolin/csrc/render/mesh/dibr_soft_mask_cuda.cu  (forward :27-184, backward :230-353)
//   kaolin/render/mesh/rasterization.py:273-371, kaolin/render/mesh/dibr.py:29-73
//
// Pipeline (forward):
//   bin_faces<count> -> scan_bins -> bin_faces<fill>
//   -> dibr_fwd2_kernel (sparse meshes on large images) | dibr_tile_fwd_kernel
//   -> soft_fwd_kernel (-> soft_tiles_fwd_kernel for leftovers)
//   * every face is turned into the exact integer pixel rectangle of the
//     reference's float bbox test and inserted (<= 4 entries) into the finest
//     level of a 16/64/256/... px bin pyramid where it spans <= 2x2 bins;
//   * one CTA per 16x16 screen tile (dibr_tile_fwd_kernel) or per 32x32 block of four
//     such tiles (dibr_fwd2_kernel) streams the bins above it into shared memory with
//     TMA bulk copies (cp.async.bulk + mbarrier, double buffered), culls them against
//     the tile, stages the surviving face records and transposes their rectangle masks
//     into per-column/row candidate bit words; each thread (one pixel) then visits
//     exactly its own rectangle hits;
//   * tiles with uncovered pixels under an enlarged (boxlen) rectangle are filed in
//     a work list; one CTA per such tile enumerates the first knum faces by index of
//     every uncovered pixel, stages each candidate face's per-face terms in shared
//     memory once, evaluates the pairs densely — one thread per (pixel, face) pair —
//     and folds them per pixel in face order.  The pairs stay in a per-tile cache
//     block for the backward pass.
// Backward: the rasterize branch walks image rows (raster_bwd_rows_kernel: one warp per
// 32 rows, per-face sums in registers flushed with vector reductions into per-face records;
// raster_bwd_kernel, a pixel-parallel scatter with a warp-level segmented reduction, when
// the shape or the workspace rules the row walk out).  The soft-mask branch is a dense
// stream over the cached pairs (soft_bwd_runs_kernel); tiles outside the cache are
// recomputed (dibr_tile_soft_bwd_kernel).
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <initializer_list>
#include <type_traits>
#include <vector>
#include <string>
#include <string.h>
#include <stdlib.h>
#include <stdint.h>

#include "../../include/dibr_b200.h"
#include "dibr_math.cuh"
#include "workspace_layout.h"

namespace {

using namespace dibr;
using namespace dibr_layout;

constexpr int kThreads = 256;
constexpr int kChunk = 256;
constexpr int kSoftCap = 1024;  // soft-mask candidates sorted per pass
constexpr int kRound = 12;      // hits a pixel contributes to one pair round
constexpr int kPairCap = kThreads * kRound;
constexpr unsigned kFull = 0xffffffffu;

// ---------------------------------------------------------------------------
// Scene description shared by all kernels (passed by value).
struct Scene {
  int B, H, W;
  int F;                  // faces per view (uniform) — 0 in packed mode
  const int64_t* first;   // packed mode: device (B+1) prefix of faces per view
  int64_t NF;             // faces in all views
  const float* xy;        // (NF,3,2)
  const float* z;         // (NF,3) or null
  int premultiplied;      // xy already scaled by multiplier
  const float* fnz;       // (NF) validity: value >= 0     (nullable)
  const uint8_t* valid;   // (NF) validity: non-zero       (nullable)
  const float* bbox_tight;  // (NF,4) given tight bboxes    (nullable -> min/max)
  const float* bbox_large;  // (NF,4) given enlarged bboxes (nullable -> min/max -/+ margin)
  float multiplier, margin;
  PixelGrid grid;
  int L;
  int ntx[kMaxLevels], nty[kMaxLevels], bin_base[kMaxLevels];
  int NB;                 // bins per view (all levels)
  int* cnt;               // [2][B][NB] (+ pool_ctr right behind it: one memset clears both)
  int* off;               // [2][B][NB]
  int4* entries;          // [2][4*NF]  {face, x_lo|x_hi<<16, y_lo|y_hi<<16, 0}
  // soft-mask hit cache: what the reference keeps as 13*knum bytes for EVERY pixel
  // (close_face_{prob,idx,dist_type}) is kept only for tiles that have hits
  int pool_tiles;         // capacity in tiles (0 = disabled)
  int pool_K;             // knum the blocks are sized for (block = 3 * 256*K words)
  int* pool_ctr;          // [1] blocks handed out
  int4* pool_hdr;         // [pool_tiles] {b, tx, ty, hits}
  uint32_t* pool_data;    // [pool_tiles][3][256*K]: face | prob bits | lx|ly<<4|(dist_type)<<8
  int* fb_ctr;            // [1] tiles whose hits did not fit the cache (recomputed in backward)
  int* fb_list;           // [B*nty*ntx] their linear tile ids
  int* tile_cnt;          // [B*nty*ceil(ntx/32)] bit per 16x16 tile: an enlarged face rectangle overlaps it (count pass)
  int* view_flag;         // [B] the view has an enlarged rectangle too big to count per tile
  int* band_ctr;          // [1] tiles with uncovered pixels under some enlarged face rectangle
  int* band_list;         // [B*nty*ntx][kBandRec] work list of the soft-mask kernels: per tile
                          //   {linear tile id, 8 x uncovered-pixel ballot, 6 x (large-bin offset, size), pad}
};

// ---------------------------------------------------------------------------
// Per-kernel timing for bench.py's roofline table (dibr_b200_trace_begin/_end):
// THREAD-LOCAL state, so the library stays re-entrant; when a trace is open on the
// calling thread every kernel launch is bracketed by a pair of CUDA events on the
// launch stream.  Off (the default) it costs one thread-local load per launch.
struct TraceState {
  bool on = false;
  int used = 0;
  std::vector<cudaEvent_t> pool;
  std::vector<const char*> names;
};
thread_local TraceState g_trace;

struct Span {
  cudaStream_t st;
  bool on;
  Span(const char* name, cudaStream_t st_) : st(st_), on(g_trace.on) {
    if (!on) return;
    TraceState& t = g_trace;
    while ((int)t.pool.size() < t.used + 2) {
      cudaEvent_t e;
      if (cudaEventCreate(&e) != cudaSuccess) { on = false; return; }
      t.pool.push_back(e);
    }
    t.names.push_back(name);
    cudaEventRecord(t.pool[t.used], st);
  }
  ~Span() {
    if (!on) return;
    cudaEventRecord(g_trace.pool[g_trace.used + 1], st);
    g_trace.used += 2;
  }
};

// ---------------------------------------------------------------------------
// PTX helpers: mbarrier + 1-D bulk TMA (global -> shared).
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes,
                                            unsigned long long* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// ---------------------------------------------------------------------------
// Face -> view lookup and face loading.
__device__ __forceinline__ void face_view(const Scene& s, int64_t i, int& b, int64_t& fbase) {
  if (s.first) {
    int lo = 0, hi = s.B;  // first[lo] <= i < first[hi]
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (__ldg(s.first + mid) <= i) lo = mid; else hi = mid;
    }
    b = lo;
    fbase = __ldg(s.first + lo);
  } else {
    b = (int)(i / s.F);
    fbase = (int64_t)b * s.F;
  }
}
__device__ __forceinline__ int64_t view_fbase(const Scene& s, int b) {
  return s.first ? __ldg(s.first + b) : (int64_t)b * s.F;
}

// xy of global face g, multiplied exactly as `face_vertices_image * multiplier`
// (rasterization.py:320, dibr.py:32): one fp32 multiply per coordinate.
__device__ __forceinline__ void load_xy(const Scene& s, int64_t g, float v[6]) {
  const float2* p = reinterpret_cast<const float2*>(s.xy + g * 6);
  const float2 a = __ldg(p), b = __ldg(p + 1), c = __ldg(p + 2);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y;
  if (!s.premultiplied) {
#pragma unroll
    for (int i = 0; i < 6; i++) v[i] = fmul(v[i], s.multiplier);
  }
}

// ---------------------------------------------------------------------------
// Binning: one thread per face; pass 1 counts, pass 2 fills (unordered inside a
// bin; consumers that need index order sort their culled candidates).
// Faces that are neighbours in the index buffer are neighbours on screen, so at any
// moment the whole GPU increments the same few bin counters, and same-address L2
// atomics serialise at the full read-modify-write latency.  The counters are therefore aggregated twice
// before they reach L2: lanes of a warp that hit the same bin are found with
// match.any, and the warp leaders merge into a per-CTA shared-memory hash table;
// one global atomic per (CTA, distinct bin) is issued by a separate thread each, so
// their round trips overlap.  The entries of a patch land contiguously.
constexpr int kBinThreadsAgg = 512;    // aggregating CTAs: big, so that a CTA merges more
constexpr int kBinThreadsPlain = 256;  // plain-atomics CTAs: small
constexpr int kBinHT = 4096;           // >= kBinThreadsAgg * 8 targets: the table always fits
constexpr uint32_t kBinEmpty = 0xffffffffu;

struct BinSmem {
  uint32_t keys[kBinHT];   // counter index (set, view, bin)
  int vals[kBinHT];        // faces of this CTA in the bin; after the flush: where they go
};

struct BinSpan { int l, bx0, bx1, by0, by1; bool has; };

__device__ __forceinline__ BinSpan bin_span(const Scene& s, const PixRect& r, bool has) {
  BinSpan sp;
  sp.has = has && r.x_hi > r.x_lo && r.y_hi > r.y_lo;
  sp.l = 0; sp.bx0 = 0; sp.bx1 = -1; sp.by0 = 0; sp.by1 = -1;
  if (sp.has) {
    for (;; ++sp.l) {
      const int sh = 4 + 2 * sp.l;
      sp.bx0 = r.x_lo >> sh; sp.bx1 = (r.x_hi - 1) >> sh;
      sp.by0 = r.y_lo >> sh; sp.by1 = (r.y_hi - 1) >> sh;
      if ((sp.bx1 - sp.bx0 <= 1 && sp.by1 - sp.by0 <= 1) || sp.l == s.L - 1) break;
    }
  }
  return sp;
}

// Registers the <= 2x2 bins of one face in the CTA table; where[k] = (table slot << 16) | rank
// inside the CTA, or -1.  Called by all lanes of the warp.
__device__ __forceinline__ void bin_insert(const Scene& s, BinSmem& sm, int set, int b, const BinSpan& sp,
                                           int (&where)[4]) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int bx = sp.bx0 + (k & 1), by = sp.by0 + (k >> 1);
    const bool on = sp.has && bx <= sp.bx1 && by <= sp.by1;
    const unsigned act = __ballot_sync(kFull, on);
    where[k] = -1;
    if (!on) continue;
    const uint32_t ci = (uint32_t)((set * s.B + b) * s.NB + s.bin_base[sp.l] + by * s.ntx[sp.l] + bx);
    const unsigned peers = __match_any_sync(act, ci);
    const int leader = __ffs(peers) - 1;
    int w = 0;
    if (lane == leader) {
      uint32_t h = (ci * 2654435761u) >> 20;
      while (true) {
        const uint32_t prev = atomicCAS(&sm.keys[h], kBinEmpty, ci);
        if (prev == kBinEmpty || prev == ci) break;
        h = (h + 1) & (kBinHT - 1);
      }
      w = (int)(h << 16) | atomicAdd(&sm.vals[h], __popc(peers));
    }
    w = __shfl_sync(peers, w, leader);
    where[k] = w + __popc(peers & ((1u << lane) - 1u));
  }
}

// Face i's multiplied xy, and in which sets it may go.  A face with a NaN among its nine
// coordinates goes into neither set (live = false): it never wins a pixel and is never a soft-mask
// candidate, so every later step sees the scene without it (DESIGN.md, NaN vertices).  The min / max
// of face_set_span drop a NaN, and the per-pixel tests pass one.  valid: live and not culled.
struct FaceState { float v[6]; bool live, valid; };

__device__ __forceinline__ FaceState face_state(const Scene& s, int64_t i, bool in_range) {
  FaceState fs;
  float* v = fs.v;
  load_xy(s, i, v);
  bool tainted = isnan(v[0]) || isnan(v[1]) || isnan(v[2]) || isnan(v[3]) || isnan(v[4]) || isnan(v[5]);
  if (s.z) tainted = tainted || isnan(__ldg(s.z + 3 * i)) || isnan(__ldg(s.z + 3 * i + 1)) || isnan(__ldg(s.z + 3 * i + 2));
  fs.live = in_range && !tainted;
  fs.valid = fs.live;
  if (s.fnz) fs.valid = fs.valid && __ldg(s.fnz + i) >= 0.f;
  if (s.valid) fs.valid = fs.valid && (__ldg(s.valid + i) != 0);
  return fs;
}

// The pixel rectangle r and bin span sp of face i in set 0 (tight) or 1 (enlarged).
__device__ __forceinline__ void face_set_span(const Scene& s, int64_t i, int set, const FaceState& fs, PixRect& r,
                                              BinSpan& sp) {
  const float* v = fs.v;
  float xmin, ymin, xmax, ymax;
  const float* given = set ? s.bbox_large : s.bbox_tight;
  if (given) {
    const float4 bb = __ldg(reinterpret_cast<const float4*>(given) + i);
    xmin = bb.x; ymin = bb.y; xmax = bb.z; ymax = bb.w;
  } else {
    // tight: torch.min / torch.max over the 3 vertices (rasterization.py:325-327);
    // large: [min - boxlen*m, max + boxlen*m] in fp32 (dibr.py:33-39)
    xmin = fminf(fminf(v[0], v[2]), v[4]); ymin = fminf(fminf(v[1], v[3]), v[5]);
    xmax = fmaxf(fmaxf(v[0], v[2]), v[4]); ymax = fmaxf(fmaxf(v[1], v[3]), v[5]);
    if (set) { xmin = fsub(xmin, s.margin); ymin = fsub(ymin, s.margin); xmax = fadd(xmax, s.margin); ymax = fadd(ymax, s.margin); }
  }
  r = bbox_to_rect(s.grid, xmin, ymin, xmax, ymax);
  sp = bin_span(s, r, set ? fs.live : fs.valid);
}

// AGG = false (sparse meshes, a few faces per tile): plain atomics, no table.
template <bool FILL, bool AGG>
__global__ void __launch_bounds__(AGG ? kBinThreadsAgg : kBinThreadsPlain, AGG ? 2 : 4)
bin_faces_kernel(Scene s, int sets) {
  constexpr int kBinThreads = AGG ? kBinThreadsAgg : kBinThreadsPlain;
  __shared__ typename std::conditional<AGG, BinSmem, int>::type sm;
  const int tid = threadIdx.x;
  if constexpr (AGG) {
    for (int t = tid; t < kBinHT; t += kBinThreads) { sm.keys[t] = kBinEmpty; sm.vals[t] = 0; }
    __syncthreads();
  }
  int64_t i = (int64_t)blockIdx.x * kBinThreads + tid;
  const bool in_range = i < s.NF;
  if (!in_range) i = s.NF - 1;
  int b; int64_t fbase;
  face_view(s, i, b, fbase);
  const int f = (int)(i - fbase);
  const FaceState fs = face_state(s, i, in_range);
  const bool live = fs.live;
  PixRect r[2];
  BinSpan sp[2];
  int where[2][4];
#pragma unroll
  for (int set = 0; set < 2; ++set) {
    sp[set].has = false;
    if (!((sets >> set) & 1)) continue;
    face_set_span(s, i, set, fs, r[set], sp[set]);
    bool aggregated = false;
    if constexpr (AGG) {
      const bool small = sp[set].bx1 - sp[set].bx0 <= 1 && sp[set].by1 - sp[set].by0 <= 1;
      aggregated = __all_sync(kFull, small);
      if (aggregated) bin_insert(s, sm, set, b, sp[set], where[set]);
    }
    if (!aggregated) {
      // (also: a warp with a face of the coarsest level spanning more than 2x2 bins)
#pragma unroll
      for (int k = 0; k < 4; ++k) where[set][k] = -1;
      if (sp[set].has) {
        const int4 e = make_int4(f, r[set].x_lo | (r[set].x_hi << 16), r[set].y_lo | (r[set].y_hi << 16), 0);
        for (int by = sp[set].by0; by <= sp[set].by1; ++by)
          for (int bx = sp[set].bx0; bx <= sp[set].bx1; ++bx) {
            const size_t ci = ((size_t)set * s.B + b) * s.NB + s.bin_base[sp[set].l] + by * s.ntx[sp[set].l] + bx;
            const int pos = atomicAdd(s.cnt + ci, 1);
            if (FILL) s.entries[(size_t)set * 4 * s.NF + 4 * fbase + s.off[ci] + pos] = e;
          }
      }
    }
  }
  if (!FILL && (sets & 2) && live && r[1].x_hi > r[1].x_lo && r[1].y_hi > r[1].y_lo) {
    // which 16x16 tiles can see this face in the soft mask (filters the soft-mask work
    // list): one bit per tile, a row of tiles per 32-bit word, so a face ORs one word per
    // tile row
    const int tx0 = r[1].x_lo >> 4, tx1 = (r[1].x_hi - 1) >> 4, ty0 = r[1].y_lo >> 4, ty1 = (r[1].y_hi - 1) >> 4;
    const int w0 = tx0 >> 5, w1 = tx1 >> 5, nw = (s.ntx[0] + 31) >> 5;
    if ((ty1 - ty0 + 1) * (w1 - w0 + 1) <= 64) {
      for (int w = w0; w <= w1; ++w) {
        const int lo = max(tx0 - (w << 5), 0), hi = min(tx1 - (w << 5), 31);
        const uint32_t m = (0xffffffffu >> (31 - hi)) & (0xffffffffu << lo);
        // a (possibly stale) L1 copy that already shows the bits saves the reduction: the
        // faces of a patch all set the same words, and same-address reductions serialise
        for (int t0 = ty0; t0 <= ty1; t0 += 4) {
          int* p = s.tile_cnt + ((size_t)b * s.nty[0] + t0) * nw + w;
          uint32_t have[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) have[j] = t0 + j <= ty1 ? (uint32_t)__ldca(p + (size_t)j * nw) : m;
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if ((have[j] & m) != m) atomicOr(p + (size_t)j * nw, (int)m);
        }
      }
    } else {
      atomicOr(s.view_flag + b, 1);
    }
  }
  if constexpr (AGG) {
    __syncthreads();
    // one global atomic per distinct bin of this CTA, each from its own thread
    for (int t = tid; t < kBinHT; t += kBinThreads) {
      const uint32_t ci = sm.keys[t];
      if (ci != kBinEmpty) {
        const int pos = atomicAdd(s.cnt + ci, sm.vals[t]);
        if (FILL) sm.vals[t] = pos + s.off[ci];
      }
    }
    if (!FILL) return;
    __syncthreads();
#pragma unroll
    for (int set = 0; set < 2; ++set) {
      const int4 e = make_int4(f, r[set].x_lo | (r[set].x_hi << 16), r[set].y_lo | (r[set].y_hi << 16), 0);
      int4* dst = s.entries + (size_t)set * 4 * s.NF + 4 * fbase;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int w = where[set][k];
        if (sp[set].has && w >= 0) dst[sm.vals[w >> 16] + (w & 0xffff)] = e;
      }
    }
  }
}

// Count pass in view-owned chunks (sparse meshes whose view's counters fit in shared memory): CTA
// (c, b) counts faces [c * chunk, (c + 1) * chunk) of view b into a shared copy of the view's bin
// counters and soft-mask tile bitmask words, then flushes one reduction per non-zero counter and word.
// The hot counters of a screen patch thus see one global reduction per CTA instead of one atomic per
// face.
// Shared memory: the requested sets' counters [nsets][NB], then (with the enlarged set) the view's
// nty * ceil(ntx / 32) bitmask words and its view_flag word.
constexpr int kBinChunkThreads = 256;
constexpr int kBinChunkMaxPerThread = 8;            // faces per thread, at most
constexpr int kBinChunkTargetCtas = 2 * 132;        // two CTAs per SM of an H100 SXM
constexpr size_t kBinChunkSmemBudget = 48 * 1024;   // no opt-in: several CTAs per SM

__host__ __device__ inline int bin_chunk_words(const Scene& s, int sets) {
  const int nsets = (sets & 1) + ((sets >> 1) & 1);
  const int bitmask = (sets & 2) ? s.nty[0] * ((s.ntx[0] + 31) >> 5) + 1 : 0;
  return nsets * s.NB + bitmask;
}

__global__ void __launch_bounds__(kBinChunkThreads) bin_count_chunk_kernel(Scene s, int sets, int chunk) {
  extern __shared__ int bin_sm[];
  const int tid = threadIdx.x;
  const int b = blockIdx.y;
  const int64_t fbase = (int64_t)b * s.F;
  const int f0 = blockIdx.x * chunk, f1 = min(f0 + chunk, s.F);
  const int nw = (s.ntx[0] + 31) >> 5;
  const int nwords = (sets & 2) ? s.nty[0] * nw : 0;
  const int total = bin_chunk_words(s, sets);
  int* const words = bin_sm + total - (nwords + 1);       // with the enlarged set only
  for (int t = tid; t < total; t += kBinChunkThreads) bin_sm[t] = 0;
  __syncthreads();
  // the shared counter of (set, bin): the sets are packed, so a single set sits at 0
  auto counter = [&](int set, const BinSpan& sp, int bx, int by) -> int* {
    return bin_sm + (sets == 3 ? set * s.NB : 0) + s.bin_base[sp.l] + by * s.ntx[sp.l] + bx;
  };
  for (int f = f0 + tid; f < f1; f += kBinChunkThreads) {
    // both sets' spans before the first shared atomic: interleaving them with the atomics measured
    // 0.14 ms instead of 0.057 ms at c4_shard (H100 80GB HBM3, 700 W)
    const int64_t i = fbase + f;
    const FaceState fs = face_state(s, i, true);
    PixRect r[2];
    BinSpan sp[2];
#pragma unroll
    for (int set = 0; set < 2; ++set) {
      sp[set].has = false;
      if ((sets >> set) & 1) face_set_span(s, i, set, fs, r[set], sp[set]);
    }
#pragma unroll
    for (int set = 0; set < 2; ++set)
      if (sp[set].has)
        for (int by = sp[set].by0; by <= sp[set].by1; ++by)
          for (int bx = sp[set].bx0; bx <= sp[set].bx1; ++bx) atomicAdd(counter(set, sp[set], bx, by), 1);
    if (nwords && fs.live && r[1].x_hi > r[1].x_lo && r[1].y_hi > r[1].y_lo) {
      // the rule of bin_faces_kernel: one bit per 16x16 tile under the enlarged rectangle, or the
      // view's flag when it covers more than 64 (tile row, word) cells
      const int tx0 = r[1].x_lo >> 4, tx1 = (r[1].x_hi - 1) >> 4, ty0 = r[1].y_lo >> 4, ty1 = (r[1].y_hi - 1) >> 4;
      const int w0 = tx0 >> 5, w1 = tx1 >> 5;
      if ((ty1 - ty0 + 1) * (w1 - w0 + 1) <= 64) {
        for (int w = w0; w <= w1; ++w) {
          const int lo = max(tx0 - (w << 5), 0), hi = min(tx1 - (w << 5), 31);
          const int m = (int)((0xffffffffu >> (31 - hi)) & (0xffffffffu << lo));
          for (int ty = ty0; ty <= ty1; ++ty)
            if ((words[ty * nw + w] & m) != m) atomicOr(&words[ty * nw + w], m);
        }
      } else {
        words[nwords] = 1;
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int set = 0; set < 2; ++set) {
    if (!((sets >> set) & 1)) continue;
    const int* c = bin_sm + (sets == 3 ? set * s.NB : 0);
    int* g = s.cnt + ((size_t)set * s.B + b) * s.NB;
    for (int t = tid; t < s.NB; t += kBinChunkThreads)
      if (c[t]) atomicAdd(g + t, c[t]);
  }
  if (nwords) {
    int* g = s.tile_cnt + (size_t)b * s.nty[0] * nw;
    for (int t = tid; t < nwords; t += kBinChunkThreads)
      if (words[t]) atomicOr(g + t, words[t]);
    if (tid == 0 && words[nwords]) atomicOr(s.view_flag + b, 1);
  }
}

// Fill pass for the shapes of bin_count_chunk_kernel: CTA (c, b) places faces [256 c, 256 c + 256) of
// view b, one per thread.  Each face takes its rank in each of its bins from a returning shared
// atomic on the view's counters (kept in registers: <= 4 per set); after a barrier one returning
// global atomic per non-zero counter claims the CTA's range of the bin, and each face writes its entry
// at off + claimed + rank.  One face per thread keeps thousands of CTAs in flight, which hides the
// latency of the claim; the entries of a bin still land in one contiguous run per CTA.  (A fill in
// the count pass's chunks of up to 2048 faces, which counted again and then handed out slots in a
// second walk over its faces, measured slower than plain atomics on an H100 80GB HBM3 at 700 W:
// 0.20 vs 0.16 ms at c4_shard; this kernel measured 0.096 ms there, 0.16 vs 0.23 ms at c3.)
__global__ void __launch_bounds__(kBinChunkThreads) bin_fill_chunk_kernel(Scene s, int sets) {
  extern __shared__ int bin_sm[];
  const int tid = threadIdx.x;
  const int b = blockIdx.y;
  const int64_t fbase = (int64_t)b * s.F;
  const int f = blockIdx.x * kBinChunkThreads + tid;
  const int ncnt = ((sets & 1) + ((sets >> 1) & 1)) * s.NB;
  for (int t = tid; t < ncnt; t += kBinChunkThreads) bin_sm[t] = 0;
  const int64_t i = fbase + min(f, s.F - 1);
  const FaceState fs = face_state(s, i, f < s.F);
  PixRect r[2];
  BinSpan sp[2];
#pragma unroll
  for (int set = 0; set < 2; ++set) {
    sp[set].has = false;
    if ((sets >> set) & 1) face_set_span(s, i, set, fs, r[set], sp[set]);
  }
  __syncthreads();
  // a span has at most 2x2 bins: the coarsest level's one bin holds the whole image
  int* c[2][4];
  int rank[2][4];
#pragma unroll
  for (int set = 0; set < 2; ++set)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int bx = sp[set].bx0 + (k & 1), by = sp[set].by0 + (k >> 1);
      c[set][k] = nullptr;
      if (sp[set].has && bx <= sp[set].bx1 && by <= sp[set].by1) {
        c[set][k] = bin_sm + (sets == 3 ? set * s.NB : 0) + s.bin_base[sp[set].l] + by * s.ntx[sp[set].l] + bx;
        rank[set][k] = atomicAdd(c[set][k], 1);
      }
    }
  __syncthreads();
#pragma unroll
  for (int set = 0; set < 2; ++set) {
    if (!((sets >> set) & 1)) continue;
    int* cs = bin_sm + (sets == 3 ? set * s.NB : 0);
    const size_t g = ((size_t)set * s.B + b) * s.NB;
    for (int t = tid; t < s.NB; t += kBinChunkThreads) {
      const int n = cs[t];
      if (n) cs[t] = __ldg(s.off + g + t) + atomicAdd(s.cnt + g + t, n);
    }
  }
  __syncthreads();
#pragma unroll
  for (int set = 0; set < 2; ++set) {
    const int4 e = make_int4(f, r[set].x_lo | (r[set].x_hi << 16), r[set].y_lo | (r[set].y_hi << 16), 0);
    int4* dst = s.entries + (size_t)set * 4 * s.NF + 4 * fbase;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (c[set][k]) dst[*c[set][k] + rank[set][k]] = e;
  }
}

// Exclusive scan of the NB bin counters of one (set, view); resets the counters
// so that the fill pass can reuse them as cursors.
__global__ void __launch_bounds__(1024) scan_bins_kernel(Scene s) {
  __shared__ int warp_sums[32];
  __shared__ int carry;
  int* cnt = s.cnt + (size_t)blockIdx.x * s.NB;
  int* off = s.off + (size_t)blockIdx.x * s.NB;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < s.NB; base += 1024) {
    const int i = base + tid;
    const int v = i < s.NB ? cnt[i] : 0;
    int x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(kFull, x, d);
      if (lane >= d) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int w = warp_sums[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_up_sync(kFull, w, d);
        if (lane >= d) w += y;
      }
      warp_sums[lane] = w;
    }
    __syncthreads();
    const int excl = carry + (warp ? warp_sums[warp - 1] : 0) + x - v;
    if (i < s.NB) { off[i] = excl; cnt[i] = 0; }
    __syncthreads();
    if (tid == 1023) carry = excl + v;
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------
// Tile helpers.
__device__ __forceinline__ uint32_t tile_mask(const int4& e, int tile_x0, int tile_y0) {
  const int x_lo = e.y & 0xffff, x_hi = (int)((unsigned)e.y >> 16);
  const int y_lo = e.z & 0xffff, y_hi = (int)((unsigned)e.z >> 16);
  const int cx0 = max(x_lo - tile_x0, 0), cx1 = min(x_hi - tile_x0, kTile);
  const int cy0 = max(y_lo - tile_y0, 0), cy1 = min(y_hi - tile_y0, kTile);
  if (cx1 <= cx0 || cy1 <= cy0) return 0u;
  const uint32_t cm = ((1u << cx1) - 1u) & ~((1u << cx0) - 1u);
  const uint32_t rm = ((1u << cy1) - 1u) & ~((1u << cy0) - 1u);
  return cm | (rm << 16);
}

struct TileCtx {
  int b, tx, ty, tile_x0, tile_y0;
  int lx, ly, px, py;
  bool in_img;
  float x0, y0;
  uint32_t sel;
  int64_t fbase, pix;
};

__device__ __forceinline__ TileCtx make_tile_ctx(const Scene& s, int b, int tx, int ty) {
  TileCtx c;
  c.tx = tx; c.ty = ty; c.b = b;
  c.tile_x0 = c.tx * kTile;
  c.tile_y0 = c.ty * kTile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  c.lx = ((warp & 1) << 3) | (lane & 7);      // each warp owns an 8x4 pixel block
  c.ly = ((warp >> 1) << 2) | (lane >> 3);
  c.px = c.tile_x0 + c.lx;
  c.py = c.tile_y0 + c.ly;
  c.in_img = c.px < s.W && c.py < s.H;
  c.x0 = pix_x(s.grid, c.px);
  c.y0 = pix_y(s.grid, c.py);
  c.sel = (1u << c.lx) | (1u << (16 + c.ly));
  c.fbase = view_fbase(s, c.b);
  c.pix = ((int64_t)c.b * s.H + c.py) * s.W + c.px;
  return c;
}

// bins above tile (tx,ty) in bin set `set`
struct BinRef { const int4* ptr; int n; };
__device__ __forceinline__ BinRef tile_bin(const Scene& s, int b, int tx, int ty, int64_t fbase,
                                           int set, int l) {
  const int sh = 2 * l;
  const int bin = s.bin_base[l] + (ty >> sh) * s.ntx[l] + (tx >> sh);
  const size_t ci = ((size_t)set * s.B + b) * s.NB + bin;
  BinRef r;
  r.n = s.cnt[ci];
  r.ptr = s.entries + (size_t)set * 4 * s.NF + 4 * fbase + s.off[ci];
  return r;
}

// Shared memory of the soft-mask backward tile kernel and of the float64 kernel.
struct TileSmem {
  float4 cxy0[kChunk];                   // ax ay bx by
  float2 cxy1[kChunk];                   // cx cy
  uint32_t cmask[kChunk];                // col mask | row mask << 16 (tile local)
  int cface[kChunk];
  unsigned long long list[kSoftCap];     // (face << 32) | mask, unsorted
  unsigned long long sorted[kSoftCap];
  float acc[kChunk][6];                  // soft-mask backward per-candidate sums
  BinRef bin[2][kMaxLevels];             // the tile's bins (set, level): filled once by warp 0
  uint8_t apix[kThreads];                // compacted uncovered pixels of the tile: lx | ly << 4
  int wcount[kThreads / 32];
  int nsoft;
};

// Shared memory of the rasterizing tile kernel (a subset: 4-5 CTAs more per SM).
struct RasterSmem {
  int4 stage[2][kChunk];
  float4 cxy0[kChunk];
  float4 cz[kChunk];
  float2 cxy1[kChunk];
  int cface[kChunk];
  uint32_t colbits[kChunk / 32][16];     // [group of 32 candidates][tile column] -> candidate bits
  uint32_t rowbits[kChunk / 32][16];     // [group][tile row]
  unsigned long long bar[2];
  BinRef bin[2][kMaxLevels];
  int any_uncovered, warps_done;
  unsigned uncmask[kThreads / 32];
};

// Transposes the tile-local rectangle masks of the 32 candidates held by a warp
// (one per lane) into per-column / per-row candidate bit words: a pixel (lx, ly)
// is inside candidate j's rectangle  <=>  bit j of colbits[g][lx] & rowbits[g][ly].
// Every pixel then walks exactly its own rectangle hits (ffs), lane-privately.
__device__ __forceinline__ void store_bit_matrix(uint32_t m, uint32_t (*colbits)[16], uint32_t (*rowbits)[16],
                                                 int g) {
  const int lane = threadIdx.x & 31;
  uint32_t mine = 0;
  if (__any_sync(kFull, m != 0)) {
#pragma unroll
    for (int b = 0; b < 32; ++b) {
      const uint32_t r = __ballot_sync(kFull, (m >> b) & 1u);
      if (lane == b) mine = r;
    }
  }
  if (lane < 16) colbits[g][lane] = mine; else rowbits[g][lane - 16] = mine;
}

// Lanes 0..L-1 / 8..8+L-1 of warp 0 look up the tight / large bins of the tile.
template <typename SM>
__device__ __forceinline__ void load_bin_table(const Scene& s, const TileCtx& c, SM& sm) {
  const int tid = threadIdx.x;
  if (tid < 16) {
    const int set = tid >> 3, l = tid & 7;
    if (l < kMaxLevels) {
      BinRef r; r.ptr = nullptr; r.n = 0;
      if (l < s.L) r = tile_bin(s, c.b, c.tx, c.ty, c.fbase, set, l);
      sm.bin[set][l] = r;
    }
  }
}

// ---------------------------------------------------------------------------
// Rasterization of one tile: walks the "tight" bins of every level.
struct RasterOut { float z, w0, w1, w2; int f; };

template <typename SM>
__device__ __forceinline__ void raster_tile(const Scene& s, const TileCtx& c, const RasterConst& rc,
                                            SM& sm, RasterOut& o) {
  const int tid = threadIdx.x;
  o.z = -INFINITY; o.f = -1; o.w0 = o.w1 = o.w2 = 0.f;

  // The (<= 6) tight bins above the tile form one virtual list, streamed in
  // rounds of kChunk entries: one mbarrier per round, one bulk copy per level piece.
  int nl[kMaxLevels];
  int total = 0;
#pragma unroll
  for (int l = 0; l < kMaxLevels; ++l) { nl[l] = sm.bin[0][l].n; total += nl[l]; }
  if (total == 0) return;  // uniform for the CTA
  const int nrounds = (total + kChunk - 1) / kChunk;

  auto issue = [&](int k) {  // thread 0 only
    const int lo = k * kChunk, hi = min(total, lo + kChunk);
    unsigned long long* bar = &sm.bar[k & 1];
    mbar_expect_tx(bar, (uint32_t)(hi - lo) * 16u);
    int start = 0;
#pragma unroll
    for (int l = 0; l < kMaxLevels; ++l) {
      const int a = max(lo, start), b = min(hi, start + nl[l]);
      if (b > a) tma_load_1d(&sm.stage[k & 1][a - lo], sm.bin[0][l].ptr + (a - start), (uint32_t)(b - a) * 16u, bar);
      start += nl[l];
    }
  };

  if (tid == 0) issue(0);
  for (int k = 0; k < nrounds; ++k) {
    if (tid == 0 && k + 1 < nrounds) issue(k + 1);  // buffer (k+1)&1 was released by the sync ending round k-1
    const int cnt = min(kChunk, total - k * kChunk);
    if ((tid & ~31) < cnt) mbar_wait(&sm.bar[k & 1], (uint32_t)((k >> 1) & 1));   // only the warps that read the buffer poll

    // cull against the tile, gather the face record (candidate id = position in the round)
    uint32_t m = 0;
    if (tid < cnt) {
      const int4 e = sm.stage[k & 1][tid];
      m = tile_mask(e, c.tile_x0, c.tile_y0);
      if (m) {
        const int64_t g = c.fbase + e.x;
        float v[6];
        load_xy(s, g, v);
        const float* zp = s.z + g * 3;
        sm.cxy0[tid] = make_float4(v[0], v[1], v[2], v[3]);
        sm.cxy1[tid] = make_float2(v[4], v[5]);
        sm.cz[tid] = make_float4(__ldg(zp), __ldg(zp + 1), __ldg(zp + 2), 0.f);
        sm.cface[tid] = e.x;
      }
    }
    if ((tid & ~31) < cnt) store_bit_matrix(m, sm.colbits, sm.rowbits, tid >> 5);
    __syncthreads();
    const int ngroups = (cnt + 31) >> 5;
    for (int g = 0; g < ngroups; ++g) {
      uint32_t bits = sm.colbits[g][c.lx] & sm.rowbits[g][c.ly];
      while (bits) {  // lane-private walk over this pixel's rectangle hits
        const int j = (g << 5) + __ffs(bits) - 1;
        bits &= bits - 1;
        const float4 q0 = sm.cxy0[j];
        const float2 q1 = sm.cxy1[j];
        float w0, w1, w2;
        if (!raster_weights(rc, c.x0, c.y0, q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, w0, w1, w2)) continue;
        const float4 zz = sm.cz[j];
        const float zv = raster_depth(zz.x, zz.y, zz.z, w0, w1, w2);
        const int f = sm.cface[j];
        // reference: strict '>' in ascending face order == (z, lowest index) maximum
        if (!(zv <= o.z) || (zv == o.z && f < o.f)) { o.z = zv; o.f = f; o.w0 = w0; o.w1 = w1; o.w2 = w2; }
      }
    }
    if (k + 1 < nrounds) __syncthreads();
  }
}

// ---------------------------------------------------------------------------
// Soft mask of one tile (forward) / its gradient (backward).  Candidates are the
// faces of the "large" bins whose enlarged rectangle meets the tile, visited in
// ascending face index; a pixel stops after knum hits.
template <bool FILTER_ONLY_COUNT, typename SM>
__device__ __forceinline__ int soft_collect(const Scene& s, const TileCtx& c, SM& sm, int lo, int hi) {
  const int tid = threadIdx.x, lane = tid & 31;
  if (tid == 0) sm.nsoft = 0;
  __syncthreads();
  for (int l = 0; l < s.L; ++l) {
    const BinRef bin = sm.bin[1][l];
    for (int base = 0; base < bin.n; base += kThreads) {
      const int i = base + tid;
      uint32_t m = 0; int f = 0;
      if (i < bin.n) {
        const int4 e = __ldg(bin.ptr + i);
        f = e.x;
        if (f > lo && f <= hi) m = tile_mask(e, c.tile_x0, c.tile_y0);
      }
      const unsigned vote = __ballot_sync(kFull, m != 0);
      if (vote) {
        int wbase = 0;
        if (lane == 0) wbase = atomicAdd(&sm.nsoft, __popc(vote));
        wbase = __shfl_sync(kFull, wbase, 0);
        if (!FILTER_ONLY_COUNT && m) {
          const int slot = wbase + __popc(vote & ((1u << lane) - 1u));
          if (slot < kSoftCap) sm.list[slot] = ((unsigned long long)(uint32_t)f << 32) | m;
        }
      }
    }
  }
  __syncthreads();
  const int n = sm.nsoft;
  __syncthreads();  // everyone has read the count before a following call resets it
  return n;
}

// Collects the tile's soft-mask candidates with face index in (lo, hi] into sm.list.
// Normally hi = INT_MAX takes everything; when more than kSoftCap faces remain
// (sub-pixel triangles) a prefix window in index order is taken instead: its upper end
// is guessed from the average index density and halved until it fits (1-3 counting
// passes), the caller continues with lo = hi until every pixel has its knum faces.  A
// window that comes out empty (the candidates cluster at higher indices) is moved past, so
// n = 0 always means that no candidate is left above lo.
template <typename SM>
__device__ __forceinline__ int soft_window(const Scene& s, const TileCtx& c, SM& sm, int lo, int maxf, int& hi) {
  hi = 0x7fffffff;
  int n = soft_collect<false>(s, c, sm, lo, hi);
  if (n > kSoftCap) {
    const int span = maxf - 1 - lo;  // indices lo+1 .. maxf-1
    int width = (int)(((long long)span * kSoftCap * 3) / ((long long)n * 4));
    if (width < 1) width = 1;
    while (true) {
      hi = lo + width;
      const int in_window = soft_collect<true>(s, c, sm, lo, hi);
      if (in_window == 0) { lo = hi; continue; }  // all n candidates lie above hi
      if (in_window <= kSoftCap || width == 1) break;
      width = width > 1 ? width / 2 : 1;
    }
    n = soft_collect<false>(s, c, sm, lo, hi);
  }
  return n;
}

// Sorts sm.list[0..n) by face index into sm.sorted (keys are unique: a face lives in one
// level and a tile reads one bin per level).  Small lists (the usual case) use a rank
// sort, n^2/256 compares per thread and one barrier; big lists (sub-pixel triangles,
// up to kSoftCap) a shared-memory bitonic network, log^2(n) barriers.  Ends with a barrier.
template <typename SM>
__device__ __forceinline__ void soft_sort(SM& sm, int n) {
  const int tid = threadIdx.x;
  if (n <= 320) {
    for (int j = tid; j < n; j += kThreads) {
      const unsigned long long key = sm.list[j];
      int rank = 0;
      for (int i = 0; i < n; ++i) rank += (sm.list[i] < key) ? 1 : 0;
      sm.sorted[rank] = key;
    }
    __syncthreads();
    return;
  }
  int np = 512;
  while (np < n) np <<= 1;
  for (int j = tid; j < np; j += kThreads) sm.sorted[j] = j < n ? sm.list[j] : ~0ull;
  __syncthreads();
  for (int k = 2; k <= np; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < (np >> 1); t += kThreads) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));  // lower element of the pair
        const int l = i | j;
        const unsigned long long a = sm.sorted[i], b = sm.sorted[l];
        const bool up = (i & k) == 0;
        if ((a > b) == up) { sm.sorted[i] = b; sm.sorted[l] = a; }
      }
      __syncthreads();
    }
  }
}

struct SoftFwdOut {
  float* prob; int64_t* idx; uint8_t* type;  // K-lists (nullable)
};

__device__ __forceinline__ int tile_linear(const Scene& s, const TileCtx& c) {
  return (c.b * s.nty[0] + c.ty) * s.ntx[0] + c.tx;
}

// Arguments of the forward tile kernels.
struct FwdArgs {
  Scene s;
  RasterConst rc;
  int D;
  const void* feat;         // (NF,3,D) FT
  float sigmainv; int K;
  int cache;                // fill the soft-mask hit cache
  int from_fb;              // soft_tiles_fwd_kernel: walk fb_list instead of band_list
  void* out_feat;           // (B,H,W,D) FT
  int64_t* idx; float* out_w; float* out_soft;  // idx: output if RASTER else input
  SoftFwdOut kl;
};

// Arguments of the soft-mask backward: (1) dense kernel over the hit cache; (2) the recompute
// tile kernel for the tiles the cache could not hold (fb_list) or, with no forward state, for
// every tile.  Persistent CTAs walk the work list.
struct SoftBwdArgs {
  Scene s;
  float sigmainv; int K;
  int from_list;             // 1: tiles of fb_list only; 0: every tile
  int view_begin, view_end;  // only tiles / cache blocks of these views (dibr_b200_backward_views)
  const float* grad_soft; const float* soft; const int64_t* idx;
  float* grad_xy;
};

// Compacts the uncovered pixels of the tile (`uncovered`: the calling thread's own pixel) into
// sm.apix, lx | ly << 4 in thread order, and returns their number (uniform).  The caller orders
// the apix writes with a barrier of its own.
template <typename SM>
__device__ __forceinline__ int compact_uncovered(const TileCtx& c, SM& sm, bool uncovered) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned av = __ballot_sync(kFull, uncovered);
  if (lane == 0) sm.wcount[warp] = __popc(av);
  __syncthreads();
  int before = 0, na = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    const int cw = sm.wcount[w];
    if (w < warp) before += cw;
    na += cw;
  }
  if (uncovered) sm.apix[before + __popc(av & ((1u << lane) - 1u))] = (uint8_t)(c.lx | (c.ly << 4));
  return na;
}

// The tile's block of the soft-mask hit cache (called by one thread): a slot from pool_ctr, or
// -1 when the cache is full, with the tile filed in fb_list to be recomputed in backward.
__device__ __forceinline__ int claim_cache_block(const Scene& s, const TileCtx& c) {
  int slot = atomicAdd(s.pool_ctr, 1);
  if (slot >= s.pool_tiles) {
    slot = -1;
    s.fb_list[atomicAdd(s.fb_ctr, 1)] = tile_linear(s, c);
  }
  return slot;
}

// Face-major pair offsets (warp 0): exclusive scan of the claims per candidate cnt_c[0..cn) into
// off_c, their total into npairs.
template <typename SM>
__device__ __forceinline__ void pair_offsets(SM& sm, int cn) {
  const int lane = threadIdx.x & 31;
  int v[8], sum = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) { const int j = lane * 8 + i; v[i] = j < cn ? sm.cnt_c[j] : 0; sum += v[i]; }
  int x = sum;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(kFull, x, d); if (lane >= d) x += y; }
  int run = x - sum;
#pragma unroll
  for (int i = 0; i < 8; ++i) { const int j = lane * 8 + i; if (j < cn) sm.off_c[j] = run; run += v[i]; }
  if (lane == 31) sm.npairs = x;
}

// Soft-mask gradient of one tile, recomputed from the large bins.  `uncovered` is the calling
// thread's own pixel; the uncovered pixels of the tile are first compacted so that the expensive
// per-(pixel, face) distance work runs on densely packed warps (thread t owns the t-th uncovered
// pixel).
__device__ __forceinline__ void soft_tile_bwd(const SoftBwdArgs& a, const TileCtx& c, TileSmem& sm, bool uncovered) {
  const Scene& s = a.s;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int na = compact_uncovered(c, sm, uncovered);
  if (na == 0) return;  // uniform
  for (int i = tid; i < kChunk * 6; i += kThreads) (&sm.acc[0][0])[i] = 0.f;
  __syncthreads();
  // thread t now owns the t-th uncovered pixel
  const bool active = tid < na;
  int lx = 0, ly = 0;
  if (active) { const int p = sm.apix[tid]; lx = p & 15; ly = p >> 4; }
  const int px = c.tile_x0 + lx, py = c.tile_y0 + ly;
  const float x0 = pix_x(s.grid, px), y0 = pix_y(s.grid, py);
  const uint32_t sel = (1u << lx) | (1u << (16 + ly));
  const int64_t pix = ((int64_t)c.b * s.H + py) * s.W + px;
  float dLdp = 0.f, soft_saved = 0.f;
  if (active) { dLdp = a.grad_soft[pix]; soft_saved = a.soft[pix]; }

  int kid = 0;
  const int maxf = s.first ? (int)(__ldg(s.first + c.b + 1) - c.fbase) : s.F;
  int lo = -1;
  while (true) {
    int hi;
    int n = soft_window(s, c, sm, lo, maxf, hi);
    soft_sort(sm, n);  // by face index
    bool all_done = false;
    for (int c0 = 0; c0 < n && !all_done; c0 += kChunk) {
      const int cn = min(kChunk, n - c0);
      if (tid < cn) {
        const unsigned long long key = sm.sorted[c0 + tid];
        const int f = (int)(key >> 32);
        float v[6];
        load_xy(s, c.fbase + f, v);
        sm.cxy0[tid] = make_float4(v[0], v[1], v[2], v[3]);
        sm.cxy1[tid] = make_float2(v[4], v[5]);
        sm.cmask[tid] = (uint32_t)key;
        sm.cface[tid] = f;
      }
      __syncthreads();
      if (warp * 32 < na) {  // warps that own no uncovered pixel have nothing to do
        for (int j = 0; j < cn; ++j) {
          const bool hit = active && kid < a.K && ((sm.cmask[j] & sel) == sel);
          float g[6];
          if (hit) {
            const float4 q0 = sm.cxy0[j];
            const float2 q1 = sm.cxy1[j];
            const float v[6] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y};
            int edgeid;
            const float d2 = soft_min_dist(x0, y0, v, s.multiplier, edgeid);
            const float prob = soft_prob(d2, a.sigmainv, s.multiplier);
            soft_backward_terms(x0, y0, v, edgeid, prob, soft_saved, dLdp, a.sigmainv, s.multiplier, g);
            ++kid;
          }
          if (__any_sync(kFull, hit)) {
#pragma unroll
            for (int q = 0; q < 6; ++q) {
              float x = hit ? g[q] : 0.f;
#pragma unroll
              for (int d = 16; d > 0; d >>= 1) x += __shfl_xor_sync(kFull, x, d);
              if (lane == 0 && x != 0.f) atomicAdd(&sm.acc[j][q], x);
            }
          }
        }
      }
      all_done = __syncthreads_and(!active || kid >= a.K);
      if (tid < cn) {
        float* gp = a.grad_xy + (c.fbase + sm.cface[tid]) * 6;
#pragma unroll
        for (int q = 0; q < 6; ++q) {
          const float x = sm.acc[tid][q];
          if (x != 0.f) { atomicAdd(gp + q, x); sm.acc[tid][q] = 0.f; }
        }
      }
      __syncthreads();
    }
    if (hi == 0x7fffffff || all_done) break;
    lo = hi;
  }
}

// ---------------------------------------------------------------------------
// Soft mask forward of one tile, pair-parallel.  The uncovered pixels are
// compacted; in rounds, every pixel claims its next (<= kRound) faces in ascending
// index (respecting knum) straight from its hit bit words, the claimed (pixel, face)
// pairs are laid out face-major in shared memory, ALL 256 threads evaluate the
// expensive distance/probability of one pair each, and finally every pixel folds
// its own results in order — the same sequence of fp32/fp64 operations per pixel as
// the reference's sequential loop, with the work spread over every lane.
struct SoftSmem {
  unsigned long long list[kSoftCap];     // (face << 32) | mask, unsorted
  unsigned long long sorted[kSoftCap];
  float4 cxy0[kChunk];
  float2 cxy1[kChunk];
  int cface[kChunk];
  uint32_t colbits[kChunk / 32][16];
  uint32_t rowbits[kChunk / 32][16];
  int cnt_c[kChunk];                     // claims per face in this round
  int off_c[kChunk];                     // face-major pair offsets
  float res_prob[kPairCap];
  uint16_t claim[kThreads][kRound];      // per pixel: (face | pos << 8), then the pair slot
  uint8_t pair_cand[kPairCap];
  uint8_t pair_pix[kPairCap];
  uint8_t res_type[kPairCap];
  uint8_t apix[kThreads];
  BinRef bin[2][kMaxLevels];
  int wcount[kThreads / 32];
  int nsoft, nent, pool_slot, npairs;
};

template <bool KLISTS>
__device__ __forceinline__ void soft_tile_fwd(const FwdArgs& a, const TileCtx& c, SoftSmem& sm, bool uncovered) {
  const Scene& s = a.s;
  const int K = a.K;
  const bool cache = !KLISTS && a.cache != 0;
  const int tid = threadIdx.x, warp = tid >> 5;
  const int na = compact_uncovered(c, sm, uncovered);
  if (na == 0) return;  // uniform
  __syncthreads();
  const bool active = tid < na;  // thread t owns the t-th uncovered pixel
  int lx = 0, ly = 0;
  if (active) { const int p = sm.apix[tid]; lx = p & 15; ly = p >> 4; }
  const int64_t pix = ((int64_t)c.b * s.H + (c.tile_y0 + ly)) * s.W + (c.tile_x0 + lx);

  float allprob = 1.0f;
  int kid = 0;
  const int maxf = s.first ? (int)(__ldg(s.first + c.b + 1) - c.fbase) : s.F;
  const size_t E = (size_t)256 * s.pool_K;
  uint32_t* blk = nullptr;
  bool first_window = true;
  int lo = -1;
  while (true) {
    int hi;
    int n = soft_window(s, c, sm, lo, maxf, hi);
    if (first_window) {
      first_window = false;
      if (tid == 0) {
        sm.pool_slot = cache && n > 0 ? claim_cache_block(s, c) : -1;
        sm.nent = 0;
      }
      __syncthreads();
      if (sm.pool_slot >= 0) blk = s.pool_data + (size_t)sm.pool_slot * 3 * E;
    }
    soft_sort(sm, n);  // by face index
    bool all_done = false;
    for (int c0 = 0; c0 < n && !all_done; c0 += kChunk) {
      const int cn = min(kChunk, n - c0);
      const int ngroups = (cn + 31) >> 5;
      uint32_t m = 0;
      if (tid < cn) {
        const unsigned long long key = sm.sorted[c0 + tid];
        const int f = (int)(key >> 32);
        m = (uint32_t)key;
        float v[6];
        load_xy(s, c.fbase + f, v);
        sm.cxy0[tid] = make_float4(v[0], v[1], v[2], v[3]);
        sm.cxy1[tid] = make_float2(v[4], v[5]);
        sm.cface[tid] = f;
      }
      if (warp < ngroups) store_bit_matrix(m, sm.colbits, sm.rowbits, warp);
      sm.cnt_c[tid] = 0;
      __syncthreads();
      int g = 0;              // hit word being consumed by this pixel
      uint32_t bits = active ? (sm.colbits[0][lx] & sm.rowbits[0][ly]) : 0u;
      while (true) {
        // claim the next <= kRound faces of this pixel, in index order
        int took = 0;
        if (active) {
          while (took < kRound && kid + took < K) {
            while (bits == 0 && g + 1 < ngroups) { ++g; bits = sm.colbits[g][lx] & sm.rowbits[g][ly]; }
            if (bits == 0) break;
            const int j = (g << 5) + __ffs(bits) - 1;
            bits &= bits - 1;
            const int pos = atomicAdd(&sm.cnt_c[j], 1);
            sm.claim[tid][took] = (uint16_t)(j | (pos << 8));
            ++took;
          }
        }
        if (!__syncthreads_or(took > 0)) break;
        if (warp == 0) pair_offsets(sm, cn);
        __syncthreads();
        const int T = sm.npairs;
        const int ebase = sm.nent;
        for (int i = 0; i < took; ++i) {
          const int cl = sm.claim[tid][i];
          const int j = cl & 0xff;
          const int slot = sm.off_c[j] + (cl >> 8);
          sm.pair_cand[slot] = (uint8_t)j;
          sm.pair_pix[slot] = (uint8_t)tid;
          sm.claim[tid][i] = (uint16_t)slot;
        }
        __syncthreads();
        sm.cnt_c[tid] = 0;  // for the next round (ordered by the barrier below)
        // dense evaluation: one (pixel, face) pair per thread
        for (int u = tid; u < T; u += kThreads) {
          const int j = sm.pair_cand[u];
          const int p = sm.apix[sm.pair_pix[u]];
          const int plx = p & 15, ply = p >> 4;
          const float4 q0 = sm.cxy0[j];
          const float2 q1 = sm.cxy1[j];
          const float v[6] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y};
          int edgeid;
          const float d2 = soft_min_dist(pix_x(s.grid, c.tile_x0 + plx), pix_y(s.grid, c.tile_y0 + ply), v,
                                         s.multiplier, edgeid);
          const float prob = soft_prob(d2, a.sigmainv, s.multiplier);
          sm.res_prob[u] = prob;
          sm.res_type[u] = (uint8_t)(edgeid + 1);
          if (blk != nullptr) {
            const size_t e = (size_t)ebase + u;
            blk[e] = (uint32_t)sm.cface[j];
            blk[E + e] = __float_as_uint(prob);
            blk[2 * E + e] = (uint32_t)plx | ((uint32_t)ply << 4) | ((uint32_t)(edgeid + 1) << 8);
          }
        }
        __syncthreads();
        if (tid == 0) sm.nent = ebase + T;
        // every pixel folds its own results in face order
        for (int i = 0; i < took; ++i) {
          const int slot = sm.claim[tid][i];
          const float prob = sm.res_prob[slot];
          allprob = soft_accumulate(allprob, prob);
          if (KLISTS) {
            const int64_t o = pix * K + kid;
            a.kl.prob[o] = prob; a.kl.idx[o] = sm.cface[sm.pair_cand[slot]]; a.kl.type[o] = sm.res_type[slot];
          }
          ++kid;
        }
      }
      all_done = __syncthreads_and(!active || kid >= K);
    }
    if (hi == 0x7fffffff || all_done) break;
    lo = hi;
  }
  if (active) a.out_soft[pix] = soft_finish(allprob);
  if (blk != nullptr && tid == 0) s.pool_hdr[sm.pool_slot] = make_int4(c.b, c.tx, c.ty, sm.nent);
}

// Large-set bin table of a tile from its work-list record (threads 0..5 write it).
template <typename SM>
__device__ __forceinline__ void bins_from_record(const Scene& s, const int* rec, int64_t fbase, SM& sm) {
  const int tid = threadIdx.x;
  if (tid < kMaxLevels) {
    BinRef r;
    r.n = __ldg(rec + 10 + 2 * tid);
    r.ptr = s.entries + (size_t)4 * s.NF + 4 * fbase + __ldg(rec + 9 + 2 * tid);
    sm.bin[1][tid] = r;
  }
}

__device__ __forceinline__ TileCtx tile_ctx_from_linear(const Scene& s, int t) {
  const int tiles_xy = s.ntx[0] * s.nty[0];
  const int b = t / tiles_xy;
  const int r = t - b * tiles_xy;
  const int ty = r / s.ntx[0];
  return make_tile_ctx(s, b, r - ty * s.ntx[0], ty);
}

// ---------------------------------------------------------------------------
// Feature storage type FT: float, or __nv_bfloat16 (BASELINE configs[3] "bf16 features":
// face_features, interpolated_features and their upstream gradient are bf16 in HBM; all
// arithmetic stays fp32 on the upcast values, the result is rounded once on store, and
// grad_face_features is accumulated in fp32).  Geometry is always fp32.
template <typename FT> struct Feat;
template <> struct Feat<float> {
  static __device__ __forceinline__ float ld(const float* p) { return __ldg(p); }
  static __device__ __forceinline__ float ld_stream(const float* p) { return __ldcs(p); }
  static __device__ __forceinline__ void st(float* p, float v) { *p = v; }
};
template <> struct Feat<__nv_bfloat16> {
  static __device__ __forceinline__ float ld(const __nv_bfloat16* p) { return __bfloat162float(__ldg(p)); }
  static __device__ __forceinline__ float ld_stream(const __nv_bfloat16* p) { return __bfloat162float(__ldcs(p)); }
  static __device__ __forceinline__ void st(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }
};

// Rasterize outputs of one pixel: face index, the optional weights and the interpolated features
// (zeros where no face covers the pixel).
template <typename FT>
__device__ __forceinline__ void store_raster_pixel(const FwdArgs& a, int64_t pix, int64_t fbase, const RasterOut& o) {
  a.idx[pix] = (int64_t)o.f;
  if (a.out_w) {
    float* wp = a.out_w + pix * 3;
    wp[0] = o.w0; wp[1] = o.w1; wp[2] = o.w2;
  }
  FT* fp = static_cast<FT*>(a.out_feat) + pix * a.D;
  const FT* feat = static_cast<const FT*>(a.feat);
  if (a.D == 3) {  // the DIB-R tutorial shape (uv + mask), fully unrolled
    float r[3] = {0.f, 0.f, 0.f};
    if (o.f >= 0) {
      const FT* ff = feat + (fbase + o.f) * 9;
#pragma unroll
      for (int d = 0; d < 3; ++d)
        r[d] = raster_interp(Feat<FT>::ld(ff + d), Feat<FT>::ld(ff + 3 + d), Feat<FT>::ld(ff + 6 + d),
                             o.w0, o.w1, o.w2);
    }
    Feat<FT>::st(fp, r[0]); Feat<FT>::st(fp + 1, r[1]); Feat<FT>::st(fp + 2, r[2]);
  } else if (o.f >= 0) {
    const FT* ff = feat + (fbase + o.f) * 3 * a.D;
    for (int d = 0; d < a.D; ++d)
      Feat<FT>::st(fp + d, raster_interp(Feat<FT>::ld(ff + d), Feat<FT>::ld(ff + a.D + d),
                                         Feat<FT>::ld(ff + 2 * a.D + d), o.w0, o.w1, o.w2));
  } else {
    for (int d = 0; d < a.D; ++d) Feat<FT>::st(fp + d, 0.f);
  }
}

// Files 16x16 tile (tx, ty) of view b in the soft-mask work list when an enlarged face rectangle
// can reach it.  The record carries everything the soft-mask kernels need to start without
// re-reading face_idx or the bin tables: the linear tile id, the uncovered-pixel ballots of its
// 8 warps (ballot(q) for warp q) and its large-bin table (level 0: `bin0`, levels >= 1: `bins`)
// as (offset, size) pairs.
template <typename Ballot>
__device__ __forceinline__ void file_band_tile(const Scene& s, int b, int tx, int ty, int64_t fbase, Ballot ballot,
                                               const BinRef& bin0, const BinRef* bins) {
  const int nlarge = ((__ldg(s.tile_cnt + ((size_t)b * s.nty[0] + ty) * ((s.ntx[0] + 31) >> 5) + (tx >> 5)) >> (tx & 31)) & 1) +
                     __ldg(s.view_flag + b);
  if (nlarge > 0) {
    int* rec = s.band_list + (size_t)atomicAdd(s.band_ctr, 1) * kBandRec;
    const int4* ebase = s.entries + (size_t)4 * s.NF + 4 * fbase;
    rec[0] = (b * s.nty[0] + ty) * s.ntx[0] + tx;
    for (int q = 0; q < kThreads / 32; ++q) rec[1 + q] = ballot(q);
    for (int l = 0; l < kMaxLevels; ++l) {
      const BinRef br = l == 0 ? bin0 : bins[l];
      rec[9 + 2 * l] = br.n > 0 ? (int)(br.ptr - ebase) : 0;
      rec[10 + 2 * l] = br.n;
    }
  }
}

// Soft-mask defaults of one pixel of 16x16 tile (tx, ty) (covered: 1; uncovered with no neighbour:
// 1 - 1 = 0) and its K-list padding; tiles where an uncovered pixel may lie under an enlarged face
// go to the soft-mask work list.  No CTA barrier: warps retire independently through the tile's
// shared `uncmask`, `any_uncovered` and `warps_done`, and the last one to finish files the tile.
template <bool KLISTS>
__device__ __forceinline__ void soft_defaults(const FwdArgs& a, int b, int tx, int ty, int64_t fbase, bool in_img,
                                              int64_t pix, int best_f, unsigned* uncmask, int* any_uncovered,
                                              int* warps_done, const BinRef& bin0, const BinRef* bins) {
  const bool uncovered = in_img && best_f < 0;
  if (in_img) {
    a.out_soft[pix] = uncovered ? 0.0f : 1.0f;
    if (KLISTS) {  // padding the reference gets from at::zeros / at::full(-1)
      for (int k = 0; k < a.K; ++k) {
        const int64_t o = pix * a.K + k;
        a.kl.prob[o] = 0.f; a.kl.idx[o] = -1; a.kl.type[o] = 0;
      }
    }
  }
  const int tid = threadIdx.x;
  const unsigned wv = __ballot_sync(kFull, uncovered);
  if ((tid & 31) == 0) {
    uncmask[tid >> 5] = wv;
    if (wv) atomicOr(any_uncovered, 1);
    __threadfence_block();
    if (atomicAdd(warps_done, 1) == kThreads / 32 - 1 && atomicOr(any_uncovered, 0))
      file_band_tile(a.s, b, tx, ty, fbase, [&](int q) { return (int)atomicOr(uncmask + q, 0u); }, bin0, bins);
  }
}

// ---------------------------------------------------------------------------
// Forward tile kernel.
template <bool RASTER, bool SOFT, bool KLISTS, typename FT>
__global__ void __launch_bounds__(kThreads, 6) dibr_tile_fwd_kernel(const __grid_constant__ FwdArgs a) {
  __shared__ __align__(128) RasterSmem sm;
  const Scene& s = a.s;
  const int tid = threadIdx.x;
  const TileCtx c = make_tile_ctx(s, blockIdx.z, blockIdx.x, blockIdx.y);   // grid = (tiles_x, tiles_y, views)
  if (RASTER && tid == 32) { mbar_init(&sm.bar[0], 1); mbar_init(&sm.bar[1], 1); mbar_fence_init(); }
  if (tid == 64) { sm.any_uncovered = 0; sm.warps_done = 0; }
  load_bin_table(s, c, sm);
  __syncthreads();
  int best_f;
  if (RASTER) {
    RasterOut o;
    raster_tile(s, c, a.rc, sm, o);
    best_f = o.f;
    if (c.in_img) store_raster_pixel<FT>(a, c.pix, c.fbase, o);
  } else {
    best_f = c.in_img ? (int)a.idx[c.pix] : 0;
  }
  if (SOFT)
    soft_defaults<KLISTS>(a, c.b, c.tx, c.ty, c.fbase, c.in_img, c.pix, best_f, sm.uncmask, &sm.any_uncovered,
                          &sm.warps_done, sm.bin[1][0], sm.bin[1]);
}

// ---------------------------------------------------------------------------
// Forward tile kernel, second generation.  Same results as dibr_tile_fwd_kernel; what changed
// is where the instructions go (in the first generation a large share of the instructions per 8x4
// pixel block was per-tile fixed work shared by only 8 warps):
//   * a CTA owns 2x2 screen tiles (32x32 px) and stages their candidates ONCE
//     (bin table, TMA rounds, tile cull, face gather, bit matrices); the 4 sub-tiles are
//     then rasterized one after the other with the first generation's thread -> pixel mapping, so the
//     soft-mask work list, the hit cache and every consumer keep their 16x16 tiles;
//   * a face is inserted in up to 2x2 level-0 bins; with several of them under one CTA it is
//     taken from the first of its bins inside the CTA only (integer test on its rectangle);
//   * conservative triangle-vs-block culling: while staging, each candidate gets its three
//     edge functions as AFFINE functions of the CTA-local pixel index (computed in double,
//     oriented so that inside is >= 0), with a margin that dominates the fp32 rounding of the
//     reference's own evaluation.  A warp (8x4 block) lets lane j test candidate j at the
//     block's extreme corners; candidates that are provably outside one edge at every pixel
//     of the block are dropped (8.5 -> 4.9 candidates per block on the benchmark mesh);
//   * the surviving candidates are visited in a WARP-UNIFORM loop (broadcast shared-memory
//     reads, no per-lane bit walk); the per-pixel decision is still the exact reference
//     arithmetic of raster_weights, so face_idx stays bit-exact.
constexpr int kSide = 2 * kTile;   // CTA tile of dibr_fwd2_kernel, in pixels
constexpr int kSubs = 4;           // its 16x16 sub-tiles, row-major

struct FwdSmem {
  int4 stage[2][kChunk];
  float4 cxy0[kChunk];
  float4 cz[kChunk];
  float2 cxy1[kChunk];
  int cface[kChunk];
  float4 cedge[kChunk][3];                 // per edge: {A + margin, B, C, -}: s*u_i ~ A + B*lx + C*ly
  uint32_t colbits[kChunk / 32][kSide];
  uint32_t rowbits[kChunk / 32][kSide];
  unsigned long long bar[2];
  BinRef bin0[2][kSubs];                   // level-0 bins of the sub-tiles (set, sub)
  BinRef bin[2][kMaxLevels];               // levels >= 1 (entry 0 unused)
  int any_uncovered[kSubs], warps_done[kSubs];
  unsigned uncmask[kSubs][kThreads / 32];
};

// Affine, sign-normalised edge functions of one face over a CTA tile whose pixel (0,0) has the
// centre (X0, Y0) and whose pixel pitch is (dx, -dy).  See the kernel comment for the contract:
// s*u_i(pixel) computed by the reference in fp32 is < 0 wherever A' + B*lx + C*ly < 0.
__device__ __noinline__ void make_edge_tests(const float v[6], double X0, double Y0, double dx, double dy,
                                                int side, float4 out[3]) {
  const double ax = v[0], ay = v[1], bx = v[2], by = v[3], cx = v[4], cy = v[5];
  const double n = (bx - ax) * (cy - ay) - (by - ay) * (cx - ax);   // u0 + u1 + u2, exact up to 2^-53
  const double sgn = n < 0.0 ? -1.0 : 1.0;
  const double ext_x = side * dx, ext_y = side * dy;
  const double Rx = fmax(fmax(fabs(ax - X0), fabs(bx - X0)), fabs(cx - X0)) + ext_x;
  const double Ry = fmax(fmax(fabs(ay - Y0), fabs(by - Y0)), fabs(cy - Y0)) + ext_y;
  const double coord = fabs(X0) + fabs(Y0) + ext_x + ext_y;
  const double px[3] = {bx, cx, ax}, py[3] = {by, cy, ay};          // u0: P=b,Q=c  u1: P=c,Q=a  u2: P=a,Q=b
  const double qx[3] = {cx, ax, bx}, qy[3] = {cy, ay, by};
  double A[3], B[3], C[3], marg = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double ux = py[i] - qy[i], uy = qx[i] - px[i];            // du/dx, du/dy
    A[i] = sgn * ((px[i] - X0) * (qy[i] - Y0) - (py[i] - Y0) * (qx[i] - X0));
    B[i] = sgn * ux * dx;
    C[i] = -sgn * uy * dy;
    const double m = 1.9073486328125e-06 * Rx * Ry                                  // 2^-19: fp32 products / fma
                     + 4.76837158203125e-07 * coord * (fabs(ux) + fabs(uy))          // 2^-21: pixel-centre rounding
                     + 9.5367431640625e-07 * (fabs(A[i]) + side * (fabs(B[i]) + fabs(C[i])));  // 2^-20: the block test itself
    marg = fmax(marg, m);
  }
  marg = 4.0 * marg + 1e-6;
  // the orientation must be certain and every quantity in range for the sign argument
  const bool ok = fabs(n) > 16.0 * marg && Rx < 268435456.0 && Ry < 268435456.0 && coord < 268435456.0;
#pragma unroll
  for (int i = 0; i < 3; ++i)
    out[i] = ok ? make_float4((float)(A[i] + marg), (float)B[i], (float)C[i], 0.f)
                : make_float4(INFINITY, 0.f, 0.f, 0.f);           // never culled (also NaN / Inf input)
}

#define DIBR_FWD2_MINB 4   /* H100, c4_shard: 4 CTAs/SM 0.97 ms, 5: 0.98, 6: 1.10, 8: 1.59 */
template <bool SOFT, typename FT>
__global__ void __launch_bounds__(kThreads, DIBR_FWD2_MINB) dibr_fwd2_kernel(const __grid_constant__ FwdArgs a) {
  constexpr int kPieces = kSubs + kMaxLevels - 1;
  __shared__ __align__(128) FwdSmem sm;
  const Scene& s = a.s;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.z;
  const int ctx0 = blockIdx.x * 2, cty0 = blockIdx.y * 2;   // first 16x16 tile of the CTA
  const int cta_x0 = ctx0 * kTile, cta_y0 = cty0 * kTile;
  const int64_t fbase = view_fbase(s, b);

  if (tid == 32) { mbar_init(&sm.bar[0], 1); mbar_init(&sm.bar[1], 1); mbar_fence_init(); }
  if (tid >= 64 && tid < 64 + kSubs) { sm.any_uncovered[tid - 64] = 0; sm.warps_done[tid - 64] = 0; }
  if (tid < 2 * kSubs) {
    const int set = tid / kSubs, sub = tid % kSubs;
    const int tx = ctx0 + sub % 2, ty = cty0 + sub / 2;
    BinRef r; r.ptr = nullptr; r.n = 0;
    if (tx < s.ntx[0] && ty < s.nty[0]) r = tile_bin(s, b, tx, ty, fbase, set, 0);
    sm.bin0[set][sub] = r;
  } else if (tid >= 96 && tid < 96 + 16) {
    const int set = (tid - 96) >> 3, l = (tid - 96) & 7;
    if (l < kMaxLevels) {
      BinRef r; r.ptr = nullptr; r.n = 0;
      if (l >= 1 && l < s.L) r = tile_bin(s, b, ctx0, cty0, fbase, set, l);
      sm.bin[set][l] = r;
    }
  }
  __syncthreads();

  // the tight bins above the CTA tile as one virtual list: 4 level-0 pieces, then levels 1..
  auto pn = [&](int p) { return p < kSubs ? sm.bin0[0][p].n : sm.bin[0][p - kSubs + 1].n; };
  int total = 0;
#pragma unroll
  for (int p = 0; p < kPieces; ++p) total += pn(p);
  const int nrounds = (total + kChunk - 1) / kChunk;
  int issued = 0, waited = 0;       // staging iterations (thread 0 / everyone): buffer = n & 1, parity = (n >> 1) & 1
  auto issue = [&](int k) {          // thread 0 only
    const int lo = k * kChunk, hi = min(total, lo + kChunk);
    unsigned long long* bar = &sm.bar[issued & 1];
    mbar_expect_tx(bar, (uint32_t)(hi - lo) * 16u);
    int start = 0;
#pragma unroll
    for (int p = 0; p < kPieces; ++p) {
      const int4* ptr = p < kSubs ? sm.bin0[0][p].ptr : sm.bin[0][p - kSubs + 1].ptr;
      const int np = pn(p);
      const int x = max(lo, start), y = min(hi, start + np);
      if (y > x) tma_load_1d(&sm.stage[issued & 1][x - lo], ptr + (x - start), (uint32_t)(y - x) * 16u, bar);
      start += np;
    }
    ++issued;
  };

  bool staged = false;

  // ---- CTA tiles that no valid face touches (40 % of them on the benchmark scene): the outputs are
  // constants, written as full 16-byte vectors row by row (9 stores per thread instead of 32)
  if (total == 0 && cta_x0 + kSide <= s.W && cta_y0 + kSide <= s.H && (s.W & 3) == 0 &&
      std::is_same<FT, float>::value && a.D == 3) {
    const int64_t pix_row0 = ((int64_t)b * s.H + cta_y0) * s.W + cta_x0;
    const int4 neg = make_int4(-1, -1, -1, -1);
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    constexpr int kIdxC = kSide * 8 / 16, kWC = kSide * 12 / 16, kSC = kSide * 4 / 16;   // 16-byte chunks per row
    for (int c = tid; c < kSide * kIdxC; c += kThreads) {
      const int r = c / kIdxC, ch = c - r * kIdxC;
      reinterpret_cast<int4*>(a.idx + pix_row0 + (int64_t)r * s.W)[ch] = neg;
    }
    for (int c = tid; c < kSide * kWC; c += kThreads) {
      const int r = c / kWC, ch = c - r * kWC;
      if (a.out_w) reinterpret_cast<float4*>(a.out_w + (pix_row0 + (int64_t)r * s.W) * 3)[ch] = zero;
      reinterpret_cast<float4*>(static_cast<float*>(a.out_feat) + (pix_row0 + (int64_t)r * s.W) * 3)[ch] = zero;
    }
    if (SOFT) {
      for (int c = tid; c < kSide * kSC; c += kThreads) {
        const int r = c / kSC, ch = c - r * kSC;
        reinterpret_cast<float4*>(a.out_soft + pix_row0 + (int64_t)r * s.W)[ch] = zero;   // uncovered, no neighbour yet
      }
      // every pixel is uncovered: file the sub-tiles an enlarged face can reach
      if (tid < kSubs)
        file_band_tile(s, b, ctx0 + tid % 2, cty0 + tid / 2, fbase, [](int) { return -1; }, sm.bin0[1][tid], sm.bin[1]);
    }
    return;
  }

  for (int sub = 0; sub < kSubs; ++sub) {
    const int sx = sub % 2, sy = sub / 2;
    const int tx = ctx0 + sx, ty = cty0 + sy;
    if (tx >= s.ntx[0] || ty >= s.nty[0]) continue;   // uniform: sub-tile outside the image
    const int lx = ((warp & 1) << 3) | (lane & 7);     // each warp owns an 8x4 pixel block
    const int ly = ((warp >> 1) << 2) | (lane >> 3);
    const int px = tx * kTile + lx, py = ty * kTile + ly;
    const bool in_img = px < s.W && py < s.H;
    const int64_t pix = ((int64_t)b * s.H + py) * s.W + px;
    RasterOut o;
    o.z = -INFINITY; o.f = -1; o.w0 = o.w1 = o.w2 = 0.f;
    if (total > 0) {
      const float x0 = pix_x(s.grid, px), y0 = pix_y(s.grid, py);
      const int clx = sx * kTile + lx, cly = sy * kTile + ly;
      const float fbx0 = (float)(sx * kTile + ((warp & 1) << 3)), fbx1 = fbx0 + 7.f;
      const float fby0 = (float)(sy * kTile + ((warp >> 1) << 2)), fby1 = fby0 + 3.f;
      for (int k = 0; k < nrounds; ++k) {
        const int cnt = min(kChunk, total - k * kChunk);
        if (!(staged && nrounds == 1)) {
          // ---- stage round k: TMA -> cull against the CTA tile -> face records, edge tests, bit matrices
          if (tid == 0) {
            if (k == 0) issue(0);
            if (k + 1 < nrounds) issue(k + 1);   // its buffer was released by the barrier ending round k-1
          }
          const int buf = waited & 1;
          // only the warps that read the landing buffer poll the mbarrier; the others go
          // straight to the CTA barrier below and sleep there (256 polling threads cost 5 % of
          // the kernel's instructions in the first version)
          if ((tid & ~31) < cnt) mbar_wait(&sm.bar[buf], (uint32_t)((waited >> 1) & 1));
          ++waited;
          uint32_t cm = 0, rm = 0;
          if (tid < cnt) {
            const int4 e = sm.stage[buf][tid];
            const int x_lo = e.y & 0xffff, x_hi = (int)((unsigned)e.y >> 16);
            const int y_lo = e.z & 0xffff, y_hi = (int)((unsigned)e.z >> 16);
            // level-0 pieces: the face is also in the neighbouring bins it spans; take it from
            // the first of its bins inside this CTA only
            bool take = true;
            const int vi = k * kChunk + tid;
            int start = 0;
#pragma unroll
            for (int p = 0; p < kSubs; ++p) {
              const int np = pn(p);
              if (vi >= start && vi < start + np)
                take = (ctx0 + p % 2) == max(x_lo >> 4, ctx0) && (cty0 + p / 2) == max(y_lo >> 4, cty0);
              start += np;
            }
            if (take) {
              const int cx0 = max(x_lo - cta_x0, 0), cx1 = min(x_hi - cta_x0, kSide);
              const int cy0 = max(y_lo - cta_y0, 0), cy1 = min(y_hi - cta_y0, kSide);
              if (cx1 > cx0 && cy1 > cy0) {
                cm = (uint32_t)(((1ull << cx1) - 1ull) & ~((1ull << cx0) - 1ull));
                rm = (uint32_t)(((1ull << cy1) - 1ull) & ~((1ull << cy0) - 1ull));
              }
            }
            if (cm) {
              const int64_t g = fbase + e.x;
              float v[6];
              load_xy(s, g, v);
              const float* zp = s.z + g * 3;
              sm.cxy0[tid] = make_float4(v[0], v[1], v[2], v[3]);
              sm.cxy1[tid] = make_float2(v[4], v[5]);
              sm.cz[tid] = make_float4(__ldg(zp), __ldg(zp + 1), __ldg(zp + 2), 0.f);
              sm.cface[tid] = e.x;
              float4 et[3];
              make_edge_tests(v, (double)pix_x(s.grid, cta_x0), (double)pix_y(s.grid, cta_y0),
                              2.0 * (double)s.grid.inv_w, 2.0 * (double)s.grid.inv_h, kSide, et);
              sm.cedge[tid][0] = et[0]; sm.cedge[tid][1] = et[1]; sm.cedge[tid][2] = et[2];
            }
          }
          if ((tid & ~31) < cnt) {
            // transpose the rectangle masks of this warp's 32 candidates into per-column / per-row words
            const int g = tid >> 5;
            if (__any_sync(kFull, cm != 0)) {
              uint32_t mine_c = 0, mine_r = 0;
#pragma unroll
              for (int q = 0; q < kSide; ++q) {
                const uint32_t c = __ballot_sync(kFull, (cm >> q) & 1u);
                const uint32_t r = __ballot_sync(kFull, (rm >> q) & 1u);
                if (lane == (q & 31)) { mine_c = c; mine_r = r; }
              }
              if (lane < kSide) { sm.colbits[g][lane] = mine_c; sm.rowbits[g][lane] = mine_r; }
            } else if (lane < kSide) {
              sm.colbits[g][lane] = 0; sm.rowbits[g][lane] = 0;
            }
          }
          __syncthreads();
        }
        // ---- rasterize this sub-tile against the staged round
        const int ngroups = (cnt + 31) >> 5;
        for (int g = 0; g < ngroups; ++g) {
          const uint32_t mybits = sm.colbits[g][clx] & sm.rowbits[g][cly];
          const uint32_t uni = __reduce_or_sync(kFull, mybits);   // candidates whose rectangle meets the block
          if (!uni) continue;
          bool keep = false;
          if ((uni >> lane) & 1u) {                                 // lane j: candidate j against the block's corners
            const float4 e0 = sm.cedge[(g << 5) + lane][0], e1 = sm.cedge[(g << 5) + lane][1],
                         e2 = sm.cedge[(g << 5) + lane][2];
            const float h0 = e0.x + fmaxf(e0.y * fbx0, e0.y * fbx1) + fmaxf(e0.z * fby0, e0.z * fby1);
            const float h1 = e1.x + fmaxf(e1.y * fbx0, e1.y * fbx1) + fmaxf(e1.z * fby0, e1.z * fby1);
            const float h2 = e2.x + fmaxf(e2.y * fbx0, e2.y * fbx1) + fmaxf(e2.z * fby0, e2.z * fby1);
            keep = !(h0 < 0.f || h1 < 0.f || h2 < 0.f);
          }
          uint32_t surv = __ballot_sync(kFull, keep);
          while (surv) {                                            // warp-uniform loop
            const int jj = __ffs(surv) - 1;
            surv &= surv - 1;
            if (!((mybits >> jj) & 1u)) continue;
            const int j = (g << 5) + jj;
            const float4 q0 = sm.cxy0[j];
            const float2 q1 = sm.cxy1[j];
            float w0, w1, w2;
            if (!raster_weights(a.rc, x0, y0, q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, w0, w1, w2)) continue;
            const float4 zz = sm.cz[j];
            const float zv = raster_depth(zz.x, zz.y, zz.z, w0, w1, w2);
            const int f = sm.cface[j];
            // reference: strict '>' in ascending face order == (z, lowest index) maximum
            if (!(zv <= o.z) || (zv == o.z && f < o.f)) { o.z = zv; o.f = f; o.w0 = w0; o.w1 = w1; o.w2 = w2; }
          }
        }
        if (nrounds > 1) __syncthreads();   // the next round overwrites the staged arrays
      }
      staged = true;
    }
    if (in_img) store_raster_pixel<FT>(a, pix, fbase, o);
    if (SOFT)
      soft_defaults<false>(a, b, tx, ty, fbase, in_img, pix, o.f, sm.uncmask[sub], &sm.any_uncovered[sub],
                           &sm.warps_done[sub], sm.bin0[1][sub], sm.bin[1]);
  }
}

// Soft-mask forward over the work list (persistent CTAs).
template <bool KLISTS>
__global__ void __launch_bounds__(kThreads, 4) soft_tiles_fwd_kernel(const __grid_constant__ FwdArgs a) {
  extern __shared__ __align__(128) unsigned char soft_smem_raw[];
  SoftSmem& sm = *reinterpret_cast<SoftSmem*>(soft_smem_raw);
  const Scene& s = a.s;
  const int total = min(a.from_fb ? *s.fb_ctr : *s.band_ctr, s.ntx[0] * s.nty[0] * s.B);
  for (int w = blockIdx.x; w < total; w += gridDim.x) {
    const TileCtx c = tile_ctx_from_linear(s, a.from_fb ? s.fb_list[w] : s.band_list[(size_t)w * kBandRec]);
    __syncthreads();  // previous tile's shared state fully consumed
    load_bin_table(s, c, sm);
    __syncthreads();
    soft_tile_fwd<KLISTS>(a, c, sm, c.in_img && a.idx[c.pix] < 0);
  }
}

// ---------------------------------------------------------------------------
// Fused soft-mask forward (knum <= kSoftFwdK, hit cache available), persistent CTAs over the
// work list.  Per silhouette tile the uncovered pixels are compacted and the candidates
// collected and sorted by face index; then, per chunk of <= 256 candidates:
//   stage    each candidate's vertices and fp64 edge divisors (soft_face) in shared memory, once;
//   claim    every uncovered pixel takes its remaining faces of the chunk in index order
//            (<= knum in all; positions inside a face from shared-memory atomics);
//   lay out  the pairs face-major in the tile's cache block (pixel | candidate in the meta word);
//   evaluate one (pixel, face) pair per thread with all 256 threads, the face part read from
//            shared memory, and write face, probability and dist_type into the block;
//   fold     each pixel multiplies its probabilities of the chunk, in face order, into a register.
// Chunks and index windows come in ascending face order, so the fold is the reference's loop
// (dibr_soft_mask_cuda.cu:174-182) term for term.  Tiles that do not fit the cache go to fb_list
// and take the single-kernel path.
constexpr int kSoftFwdK = 32;  // largest knum of the fused kernel (claims per pixel and chunk)
constexpr int kRunHits = 8;    // consecutive cached pairs per thread in the run kernels

// Per-chunk face part.  The fp32 line terms of soft_face (A, B, C and their products) are
// recomputed from the vertices per pair: seven fp32 operations cost less than loading six floats.
struct SoftCand {
  float4 xy0[kChunk];        // vertices a, b
  float2 xy1[kChunk];        // vertex c
  DRecip down64[3][kChunk];  // per edge: (double)(A^2 + B^2) + eps and its reciprocal
};

struct SoftFwdSmem {
  union {
    unsigned long long list[kSoftCap];  // soft_window's candidates: dead once soft_sort is done
    SoftCand cand;                      // the current chunk
  };
  unsigned long long sorted[kSoftCap];
  uint32_t colbits[kChunk / 32][16];
  uint32_t rowbits[kChunk / 32][16];
  int cnt_c[kChunk];
  int off_c[kChunk];
  uint16_t claim[kThreads][kSoftFwdK];  // per pixel, face order: candidate | position << 8
  uint8_t apix[kThreads];
  BinRef bin[2][kMaxLevels];
  int nsoft, nent, pool_slot, npairs;
};

#define DIBR_SOFT_FWD_MINB 4   /* H100 (400 W), c4_shard: 4 CTAs/SM 0.81 ms, 3: 0.91, 5: 0.88, 6: 1.01 */
__global__ void __launch_bounds__(kThreads, DIBR_SOFT_FWD_MINB) soft_fwd_kernel(const __grid_constant__ FwdArgs a) {
  __shared__ __align__(128) SoftFwdSmem sm;
  const Scene& s = a.s;
  const int K = a.K;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int total = min(*s.band_ctr, s.ntx[0] * s.nty[0] * s.B);
  const int E = 256 * s.pool_K;   // block words per array (< 2^14): 32-bit offsets
  for (int w = blockIdx.x; w < total; w += gridDim.x) {
    // the work-list record carries the tile id, the uncovered-pixel ballots of the
    // rasterizer's 8 warps and the tile's large-bin table: one load latency, no
    // face_idx re-read, no barrier for the compaction
    const int* rec = s.band_list + (size_t)w * kBandRec;
    const TileCtx c = tile_ctx_from_linear(s, __ldg(rec));
    unsigned mymask = 0;
    int before = 0, na = 0;
#pragma unroll
    for (int q = 0; q < kThreads / 32; ++q) {
      const unsigned mq = (unsigned)__ldg(rec + 1 + q);
      if (q < warp) before += __popc(mq);
      if (q == warp) mymask = mq;
      na += __popc(mq);
    }
    __syncthreads();  // previous tile's shared state fully consumed
    bins_from_record(s, rec, c.fbase, sm);
    if ((mymask >> lane) & 1u) sm.apix[before + __popc(mymask & ((1u << lane) - 1u))] = (uint8_t)(c.lx | (c.ly << 4));
    const bool active = tid < na;  // thread t owns the t-th uncovered pixel
    int lx = 0, ly = 0;
    int kid = 0;
    float allprob = 1.0f;
    const int maxf = s.first ? (int)(__ldg(s.first + c.b + 1) - c.fbase) : s.F;
    uint32_t* blk = nullptr;
    bool first_window = true, cached = true;
    int lo = -1;
    while (true) {
      int hi;
      int n = soft_window(s, c, sm, lo, maxf, hi);
      if (first_window && active) { const int p = sm.apix[tid]; lx = p & 15; ly = p >> 4; }
      const bool alloc = first_window;
      if (first_window) {
        first_window = false;
        if (n == 0) { cached = false; break; }  // uncovered pixels, but no face near them: soft stays 0
        // cache block: one atomic, its round trip hidden behind the sort below
        if (tid == 0) {   // cache full: single-kernel path + recompute in backward
          sm.pool_slot = claim_cache_block(s, c);
          sm.nent = 0;
        }
      }
      soft_sort(sm, n);  // by face index
      if (alloc) {
        if (sm.pool_slot < 0) { cached = false; break; }  // uniform: handed over to the single-kernel path
        blk = s.pool_data + (size_t)sm.pool_slot * 3 * E;
      }
      bool all_done = false;
      for (int c0 = 0; c0 < n && !all_done; c0 += kChunk) {
        const int cn = min(kChunk, n - c0);
        const int ngroups = (cn + 31) >> 5;
        uint32_t m = 0;
        if (tid < cn) {  // face part of candidate tid, once per tile
          const unsigned long long key = sm.sorted[c0 + tid];
          m = (uint32_t)key;
          float v[6];
          load_xy(s, c.fbase + (int)(key >> 32), v);
          sm.cand.xy0[tid] = make_float4(v[0], v[1], v[2], v[3]);
          sm.cand.xy1[tid] = make_float2(v[4], v[5]);
          const SoftFace F = soft_face(v);
#pragma unroll
          for (int i = 0; i < 3; ++i) sm.cand.down64[i][tid] = F.down64[i];
        }
        if (warp < ngroups) store_bit_matrix(m, sm.colbits, sm.rowbits, warp);
        sm.cnt_c[tid] = 0;
        __syncthreads();
        // every uncovered pixel claims ALL its remaining faces of this chunk (index order, <= knum)
        int took = 0;
        if (active) {
          for (int g = 0; g < ngroups && kid + took < K; ++g) {
            uint32_t bits = sm.colbits[g][lx] & sm.rowbits[g][ly];
            while (bits && kid + took < K) {
              const int j = (g << 5) + __ffs(bits) - 1;
              bits &= bits - 1;
              const int pos = atomicAdd(&sm.cnt_c[j], 1);
              sm.claim[tid][took] = (uint16_t)(j | (pos << 8));
              ++took;
            }
          }
        }
        __syncthreads();
        if (warp == 0) pair_offsets(sm, cn);
        __syncthreads();
        const int ebase = sm.nent, T = sm.npairs;
        // pair -> (pixel, candidate) map in the meta words; the CTA reads it back after the barrier
        for (int i = 0; i < took; ++i) {
          const int cl = sm.claim[tid][i];
          const int j = cl & 0xff;
          blk[2 * E + ebase + sm.off_c[j] + (cl >> 8)] = (uint32_t)lx | ((uint32_t)ly << 4) | ((uint32_t)j << 16);
        }
        __syncthreads();
        // dense evaluation: one (pixel, face) pair per thread
#pragma unroll 1
        for (int u = tid; u < T; u += kThreads) {
          const int e = ebase + u;
          const uint32_t map = blk[2 * E + e];
          const int j = (int)(map >> 16);
          const int plx = (int)(map & 15u), ply = (int)((map >> 4) & 15u);
          const float4 q0 = sm.cand.xy0[j];
          const float2 q1 = sm.cand.xy1[j];
          const float v[6] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y};
          SoftFace F;
#pragma unroll
          for (int i = 0; i < 3; ++i) { F.e[i] = soft_edge(v, i); F.down64[i] = sm.cand.down64[i][j]; }
          int edgeid;
          const float d2 = soft_pixel_dist(pix_x(s.grid, c.tile_x0 + plx), pix_y(s.grid, c.tile_y0 + ply), v, F,
                                           s.multiplier, edgeid);
          const float prob = soft_prob(d2, a.sigmainv, s.multiplier);
          blk[e] = (uint32_t)(sm.sorted[c0 + j] >> 32);
          blk[E + e] = __float_as_uint(prob);
          blk[2 * E + e] = (map & 0xffu) | ((uint32_t)(edgeid + 1) << 8);
        }
        __syncthreads();
        // fold: each pixel multiplies its probabilities in face order, four loads in flight
        for (int i0 = 0; i0 < took; i0 += 4) {
          float p[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            if (i0 + q < took) {
              const int cl = sm.claim[tid][i0 + q];
              p[q] = __uint_as_float(blk[E + ebase + sm.off_c[cl & 0xff] + (cl >> 8)]);
            }
          }
#pragma unroll
          for (int q = 0; q < 4; ++q)
            if (i0 + q < took) allprob = soft_accumulate(allprob, p[q]);
        }
        kid += took;
        all_done = __syncthreads_and(!active || kid >= K);
        if (tid == 0) sm.nent = ebase + T;
      }
      if (hi == 0x7fffffff || all_done) break;
      lo = hi;
    }
    if (cached) {
      // the tile's coordinates again from the record: cheaper than keeping them in registers
      const TileCtx ce = tile_ctx_from_linear(s, __ldg(s.band_list + (size_t)w * kBandRec));
      if (active) a.out_soft[((int64_t)ce.b * s.H + (ce.tile_y0 + ly)) * s.W + (ce.tile_x0 + lx)] = soft_finish(allprob);
      if (tid == 0) s.pool_hdr[sm.pool_slot] = make_int4(ce.b, ce.tx, ce.ty, sm.nent);
    }
  }
}

// ---------------------------------------------------------------------------
// Soft-mask backward: the recompute tile kernel, then the dense kernel over the hit cache.
__global__ void __launch_bounds__(kThreads) dibr_tile_soft_bwd_kernel(const __grid_constant__ SoftBwdArgs a) {
  __shared__ __align__(128) TileSmem sm;
  const Scene& s = a.s;
  const int ntiles = s.ntx[0] * s.nty[0] * s.B;
  const int total = a.from_list ? min(*s.fb_ctr, ntiles) : ntiles;
  for (int w = blockIdx.x; w < total; w += gridDim.x) {
    const TileCtx c = tile_ctx_from_linear(s, a.from_list ? s.fb_list[w] : w);
    if (c.b < a.view_begin || c.b >= a.view_end) continue;   // uniform for the CTA
    __syncthreads();  // previous tile's shared state fully consumed
    load_bin_table(s, c, sm);
    __syncthreads();
    soft_tile_bwd(a, c, sm, c.in_img && a.idx[c.pix] < 0);
  }
}

// Dense soft-mask backward over the hit cache: the hits of a tile lie face-major in its cache
// block, so a thread that takes 8 CONSECUTIVE hits (two LDG.128 per array, 32 bytes per lane, 1 KB
// per warp request) sees one or two faces.  It sums the six partials of a face in registers and
// flushes them with three RED.v2 when the face changes - no match/shuffle reduction (30 SHFL per
// warp at 1 SHFL per clock per SM) and one face-vertex load per run instead of per hit.
#define DIBR_SBWD_MINB 4   /* H100, c4_shard: 4 CTAs/SM 0.34 ms, 3: 0.38, 5: 0.35, 6: 0.36 */
__global__ void __launch_bounds__(kThreads, DIBR_SBWD_MINB) soft_bwd_runs_kernel(const __grid_constant__ SoftBwdArgs a) {
  const Scene& s = a.s;
  const int used = min(*s.pool_ctr, s.pool_tiles);
  if ((int)blockIdx.x >= used) return;
  const int4 h = s.pool_hdr[blockIdx.x];  // b, tx, ty, hits
  if (h.x < a.view_begin || h.x >= a.view_end) return;
  const size_t E = (size_t)256 * s.pool_K;
  const uint32_t* blk = s.pool_data + (size_t)blockIdx.x * 3 * E;
  const int64_t fbase = view_fbase(s, h.x);
  const float inv_m = 1.0f / s.multiplier;
  const int64_t pix_tile = ((int64_t)h.x * s.H + (int64_t)h.z * kTile) * s.W + h.y * kTile;
  for (int start = threadIdx.x * kRunHits; start < h.w; start += kThreads * kRunHits) {
    const int n = min(kRunHits, h.w - start);
    uint32_t face[kRunHits], prob[kRunHits], meta[kRunHits];
    {
      const uint4* pf = reinterpret_cast<const uint4*>(blk + start);
      const uint4* pp = reinterpret_cast<const uint4*>(blk + E + start);
      const uint4* pm = reinterpret_cast<const uint4*>(blk + 2 * E + start);
      // the block is sized 256*K entries: reading the (unused) tail of the last group of 8 stays inside it
      const uint4 f0 = __ldcs(pf), f1 = __ldcs(pf + 1), p0 = __ldcs(pp), p1 = __ldcs(pp + 1);
      const uint4 m0 = __ldcs(pm), m1 = __ldcs(pm + 1);
      face[0] = f0.x; face[1] = f0.y; face[2] = f0.z; face[3] = f0.w; face[4] = f1.x; face[5] = f1.y; face[6] = f1.z; face[7] = f1.w;
      prob[0] = p0.x; prob[1] = p0.y; prob[2] = p0.z; prob[3] = p0.w; prob[4] = p1.x; prob[5] = p1.y; prob[6] = p1.z; prob[7] = p1.w;
      meta[0] = m0.x; meta[1] = m0.y; meta[2] = m0.z; meta[3] = m0.w; meta[4] = m1.x; meta[5] = m1.y; meta[6] = m1.z; meta[7] = m1.w;
    }
    int cur = -1;
    float v[6], acc[6];
#pragma unroll
    for (int j = 0; j < kRunHits; ++j) {
      if (j < n) {
        const int f = (int)face[j];
        if (f != cur) {
          if (cur >= 0) {
            float2* gx = reinterpret_cast<float2*>(a.grad_xy + (fbase + cur) * 6);
            if (acc[0] != 0.f || acc[1] != 0.f) atomicAdd(gx, make_float2(acc[0], acc[1]));
            if (acc[2] != 0.f || acc[3] != 0.f) atomicAdd(gx + 1, make_float2(acc[2], acc[3]));
            if (acc[4] != 0.f || acc[5] != 0.f) atomicAdd(gx + 2, make_float2(acc[4], acc[5]));
          }
          cur = f;
          load_xy(s, fbase + f, v);
#pragma unroll
          for (int q = 0; q < 6; ++q) acc[q] = 0.f;
        }
        const int lx = (int)(meta[j] & 15u), ly = (int)((meta[j] >> 4) & 15u);
        const int64_t pix = pix_tile + (int64_t)ly * s.W + lx;
        float g[6];
        soft_backward_terms_fast(pix_x(s.grid, h.y * kTile + lx), pix_y(s.grid, h.z * kTile + ly), v,
                                 (int)(meta[j] >> 8) - 1, __uint_as_float(prob[j]), __ldg(a.soft + pix),
                                 __ldg(a.grad_soft + pix), a.sigmainv, inv_m, g);
#pragma unroll
        for (int q = 0; q < 6; ++q) acc[q] += g[q];
      }
    }
    if (cur >= 0) {
      float2* gx = reinterpret_cast<float2*>(a.grad_xy + (fbase + cur) * 6);
      if (acc[0] != 0.f || acc[1] != 0.f) atomicAdd(gx, make_float2(acc[0], acc[1]));
      if (acc[2] != 0.f || acc[3] != 0.f) atomicAdd(gx + 1, make_float2(acc[2], acc[3]));
      if (acc[4] != 0.f || acc[5] != 0.f) atomicAdd(gx + 2, make_float2(acc[4], acc[5]));
    }
  }
}

// ---------------------------------------------------------------------------
// Rasterize backward: pixel-parallel; lanes of a warp (an 8x4 pixel block) that
// hit the same face are summed with a segmented shuffle reduction, so a face
// costs one group of atomics per warp instead of 9*D per pixel
// (rasterization_cuda.cu:272-285,376-399).
template <int N>
__device__ __forceinline__ void reduce_peers(unsigned peers, float (&v)[N]) {
  const int lane = threadIdx.x & 31;
  int rel = __popc(peers & ((1u << lane) - 1u));
  peers &= (0xfffffffeu << lane);  // peers above me
  while (__any_sync(kFull, peers)) {
    const int next = __ffs(peers);  // 1-based lane of my next peer, 0 if none
#pragma unroll
    for (int i = 0; i < N; ++i) {
      const float t = __shfl_sync(kFull, v[i], (next - 1) & 31);
      if (next) v[i] += t;
    }
    const unsigned done = __ballot_sync(kFull, rel & 1);
    peers &= ~done;
    rel >>= 1;
  }
}

// w == nullptr: the weights are recomputed from face_idx, xy * multiplier and the pixel grid, which
// reproduces the forward's bits when multiplier and eps are the forward's
struct RasterBwdArgs {
  int B, H, W, F, D;
  int ntx, nty;
  const void* grad_feat; const int64_t* idx; const float* w; const float* xy; const void* feat;  // FT
  PixelGrid grid; RasterConst rc; float multiplier;
  float* grad_xy; float* grad_feat_out;
};

template <int DT, typename FT>  // DT > 0: feature dim known at compile time; 0: runtime loop
__global__ void __launch_bounds__(kThreads, 6) raster_bwd_kernel(const __grid_constant__ RasterBwdArgs a) {
  const FT* grad_feat = static_cast<const FT*>(a.grad_feat);
  const FT* feat = static_cast<const FT*>(a.feat);
  const int tx = blockIdx.x, ty = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int px = tx * kTile + (((warp & 1) << 3) | (lane & 7));
  const int py = ty * kTile + (((warp >> 1) << 2) | (lane >> 3));
  const bool in_img = px < a.W && py < a.H;
  const int64_t pix = ((int64_t)b * a.H + py) * a.W + px;
  const int D = DT > 0 ? DT : a.D;
  // all streaming operands of the pixel are requested together (given weights and upstream
  // gradient do not depend on face_idx): one exposed HBM latency instead of two
  int f = -1;
  float w0 = 0.f, w1 = 0.f, w2 = 0.f;
  float gpre[DT > 0 ? DT : 1];
#pragma unroll
  for (int d = 0; d < (DT > 0 ? DT : 1); ++d) gpre[d] = 0.f;
  if (in_img) {
    f = (int)__ldcs(a.idx + pix);
    if (a.w) {
      const float* wp = a.w + pix * 3;
      w0 = __ldcs(wp); w1 = __ldcs(wp + 1); w2 = __ldcs(wp + 2);
    }
    if (DT > 0) {
#pragma unroll
      for (int d = 0; d < DT; ++d) gpre[d] = Feat<FT>::ld_stream(grad_feat + pix * DT + d);
    }
  }
  if (!__any_sync(kFull, f >= 0)) return;
  const bool cov = f >= 0;
  const int64_t face = (int64_t)b * a.F + (cov ? f : 0);

  RasterBwdGeom G;
  if (cov) {
    const float2* pp = reinterpret_cast<const float2*>(a.xy + face * 6);
    const float2 pa = __ldg(pp), pb = __ldg(pp + 1), pc = __ldg(pp + 2);
    const float p[6] = {pa.x, pa.y, pb.x, pb.y, pc.x, pc.y};
    if (!a.w) {
      const float m = a.multiplier;
      raster_weights_of(a.rc, pix_x(a.grid, px), pix_y(a.grid, py), fmul(p[0], m), fmul(p[1], m),
                        fmul(p[2], m), fmul(p[3], m), fmul(p[4], m), fmul(p[5], m), w0, w1, w2);
    }
    raster_backward_geom(p, w0, w1, w2, a.rc.eps, G);
  }
  // lanes without a face get unique negative keys so they never merge
  const unsigned peers = __match_any_sync(kFull, cov ? (int)f : -1 - lane);
  const bool leader = (peers & ((1u << lane) - 1u)) == 0;
  const FT* gp = grad_feat + pix * D;
  const FT* cf = feat + face * 3 * D;

  if (DT > 0) {
    float v[6 + 3 * (DT > 0 ? DT : 1)];
#pragma unroll
    for (int j = 0; j < 6; ++j) v[j] = 0.f;
#pragma unroll
    for (int d = 0; d < DT; ++d) {
      float g = 0.f;
      if (cov) {
        g = gpre[d];
        float t6[6];
        raster_backward_feature(G, g, Feat<FT>::ld(cf + d), Feat<FT>::ld(cf + DT + d), Feat<FT>::ld(cf + 2 * DT + d), t6);
#pragma unroll
        for (int j = 0; j < 6; ++j) v[j] += t6[j];
      }
      v[6 + d] = g * w0; v[6 + DT + d] = g * w1; v[6 + 2 * DT + d] = g * w2;
    }
    reduce_peers<6 + 3 * (DT > 0 ? DT : 1)>(peers, v);
    if (leader && cov) {
      float2* gx = reinterpret_cast<float2*>(a.grad_xy + face * 6);
      atomicAdd(gx, make_float2(v[0], v[1]));
      atomicAdd(gx + 1, make_float2(v[2], v[3]));
      atomicAdd(gx + 2, make_float2(v[4], v[5]));
      float* gf = a.grad_feat_out + face * 3 * DT;
#pragma unroll
      for (int j = 0; j < 3 * DT; ++j) atomicAdd(gf + j, v[6 + j]);
    }
  } else {
    float vx[6];
#pragma unroll
    for (int j = 0; j < 6; ++j) vx[j] = 0.f;
    for (int d = 0; d < D; ++d) {
      float g = 0.f;
      if (cov) {
        g = Feat<FT>::ld_stream(gp + d);
        float t6[6];
        raster_backward_feature(G, g, Feat<FT>::ld(cf + d), Feat<FT>::ld(cf + D + d), Feat<FT>::ld(cf + 2 * D + d), t6);
#pragma unroll
        for (int j = 0; j < 6; ++j) vx[j] += t6[j];
      }
      float v[3] = {g * w0, g * w1, g * w2};
      reduce_peers<3>(peers, v);
      if (leader && cov) {
        float* gf = a.grad_feat_out + face * 3 * D;
        atomicAdd(gf + d, v[0]); atomicAdd(gf + D + d, v[1]); atomicAdd(gf + 2 * D + d, v[2]);
      }
    }
    reduce_peers<6>(peers, vx);
    if (leader && cov) {
      float2* gx = reinterpret_cast<float2*>(a.grad_xy + face * 6);
      atomicAdd(gx, make_float2(vx[0], vx[1]));
      atomicAdd(gx + 1, make_float2(vx[2], vx[3]));
      atomicAdd(gx + 2, make_float2(vx[4], vx[5]));
    }
  }
}

// ---------------------------------------------------------------------------
// Rasterize backward, ROW-WALK variant (the one the fused path uses when the feature
// dim is 1..4 fp32 and the image width a multiple of 4).
//
// SHFL issues at a quarter of the FFMA rate (32 vs 128 results per clock per SM on
// sm_90, CUDA C++ Programming Guide, arithmetic instruction throughput), and a vector
// reduction RED.E.ADD.F32x4 moves four floats per lane in one instruction.  The kernel
// above spends 75 shuffles per covered warp on its segmented reduction and 12 scalar /
// v2 reductions per (warp, face) group; this one uses neither:
//   * a warp owns 32 image rows x `strip` columns; LANE = ROW.  The lane walks along its
//     row and accumulates the 6 + 3*D partial sums of the current face in REGISTERS; when
//     face_idx changes it flushes them with (6+3D+3)/4 vector reductions into a padded
//     per-face accumulator (acc[face][16] for D = 3: 64-byte records, 16-byte aligned) and
//     reloads the face constants.  No shuffles, no match, no leader election;
//   * the pixel streams (face_idx 8 B, upstream gradient 4*D B per pixel) are staged per
//     4-column slab with 16-byte cp.async (LDGSTS) into rows padded to an odd number of
//     16-byte chunks, double buffered, and read back with LDS.128 (conflict free: 8
//     consecutive rows cover the 32 banks).  6 KB of shared memory and <= 128 registers per
//     single-warp CTA keep 16 warps per SM in flight (8-column slabs needed 162 registers:
//     9 warps per SM);
//   * the barycentric weights are not read: each covered pixel recomputes its face's weights
//     with the forward's own arithmetic (raster_weights_of: same bits), from the face's
//     vertices times the multiplier, which the lane holds while it walks the face's run.
//     Weights given by the caller (the operator-level backward) are read per pixel instead;
//   * raster_bwd_finalize_kernel unpacks acc into grad_face_vertices_image /
//     grad_face_features (which therefore need no memset).
// Per-pixel arithmetic is the reference's operation tree (dibr_math.cuh,
// raster_backward_geom / _feature) with the face-constant factors hoisted; the only
// change is g * (1 / k3^2) for g / k3^2 (<= 1 ulp per term).
constexpr int kRwSlab = 4;   // columns per staged slab (= the 4-pixel block a lane reads with LDS.128)

template <int DT>
struct RwCfg {
  // rows padded to an ODD number of 16-byte chunks: 8 consecutive rows then cover all 32 banks
  static constexpr int pad_odd(int bytes) { return ((bytes / 16) & 1) ? bytes : bytes + 16; }
  static constexpr int kIdxPitch = pad_odd(kRwSlab * 8);        // 32 -> 48
  static constexpr int kAcc = face_record_floats(DT);           // floats per face record
};
// upstream-gradient rows: fp32 (16*D bytes, 16-byte chunks) or bf16 (8*D bytes; D odd -> 8-byte chunks,
// rows of 24 bytes are read with LDS.64: a half warp covers the 32 banks)
template <int DT, typename FT>
struct RwG {
  static constexpr int kRow = kRwSlab * DT * (int)sizeof(FT);
  static constexpr int kChunk = (kRow % 16) ? 8 : 16;
  static constexpr int kPitch = kChunk == 16 ? RwCfg<DT>::pad_odd(kRow) : kRow;
  static constexpr int kStage = 32 * (RwCfg<DT>::kIdxPitch + kPitch);
};
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async8(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

struct RowBwdArgs {
  int B, H, W, F, strip, jobs_x, jobs_y;
  const void* grad_feat; const int64_t* idx; const float* w; const float* xy; const void* feat;   // FT: float | bf16
  PixelGrid grid; RasterConst rc; float multiplier;   // w == nullptr: see RasterBwdArgs
  float* acc;    // [B*F][RwCfg<D>::kAcc], zeroed
  int* job_ctr;  // [1] zeroed (lives right behind the records)
};

template <int DT>
struct RowFace {          // constants of the face a lane is currently accumulating
  float ax, ay, bx, by, cx, cy;
  float mx[3], my[3];           // vertices * multiplier: the forward's raster coordinates
  float pp, n, m, q, k3, rk;
  float qk3, nk3n, ppk3n, mk3;  // q*k3, -(n*k3), -(pp*k3), m*k3  (dw1ds, dw1dt, dw2ds, dw2dt)
  float d1[DT], d2[DT];
};

template <int DT, typename FT>
__device__ __forceinline__ void row_face_load(const RowBwdArgs& a, int64_t face, RowFace<DT>& c) {
  const float2* pp = reinterpret_cast<const float2*>(a.xy + face * 6);
  const float2 pa = __ldg(pp), pb = __ldg(pp + 1), pc = __ldg(pp + 2);
  const FT* cf = static_cast<const FT*>(a.feat) + face * 3 * DT;
  float c0[DT], c1[DT], c2[DT];
#pragma unroll
  for (int d = 0; d < DT; ++d) { c0[d] = Feat<FT>::ld(cf + d); c1[d] = Feat<FT>::ld(cf + DT + d); c2[d] = Feat<FT>::ld(cf + 2 * DT + d); }
  c.ax = pa.x; c.ay = pa.y; c.bx = pb.x; c.by = pb.y; c.cx = pc.x; c.cy = pc.y;
  c.mx[0] = fmul(pa.x, a.multiplier); c.mx[1] = fmul(pb.x, a.multiplier); c.mx[2] = fmul(pc.x, a.multiplier);
  c.my[0] = fmul(pa.y, a.multiplier); c.my[1] = fmul(pb.y, a.multiplier); c.my[2] = fmul(pc.y, a.multiplier);
  c.pp = fsub(c.by, c.ay); c.n = fsub(c.cx, c.ax); c.m = fsub(c.bx, c.ax); c.q = fsub(c.cy, c.ay);
  float k3 = ffma(c.m, c.q, -fmul(c.pp, c.n));
  {
    const double e = (f2u(k3) >> 31) ? -fabs((double)a.rc.eps) : fabs((double)a.rc.eps);
    k3 = d2f(dibr::dadd((double)k3, e));
  }
  c.k3 = k3;
  c.rk = fdiv(1.0f, fmul(k3, k3));
  c.qk3 = fmul(c.q, k3); c.nk3n = -fmul(c.n, k3); c.ppk3n = -fmul(c.pp, k3); c.mk3 = fmul(c.m, k3);
#pragma unroll
  for (int d = 0; d < DT; ++d) { c.d1[d] = fsub(c1[d], c0[d]); c.d2[d] = fsub(c2[d], c0[d]); }
}

template <int DT>
__device__ __forceinline__ void row_pixel(const RowFace<DT>& c, float aw, float bw, float cw, const float* g,
                                          float (&acc)[RwCfg<DT>::kAcc]) {
  const float y0 = ffma(c.cy, cw, ffma(c.ay, aw, fmul(c.by, bw)));
  const float x0 = ffma(c.cx, cw, ffma(c.ax, aw, fmul(c.bx, bw)));
  const float t = fsub(y0, c.ay), s = fsub(x0, c.ax);
  const float k1 = ffma(c.q, s, -fmul(c.n, t));
  const float k2 = ffma(c.m, t, -fmul(c.pp, s));
  const float tk3 = fmul(t, c.k3), sk3 = fmul(s, c.k3);
  const float dw1dm = -fmul(c.q, k1);
  const float dw2dm = ffma(-c.q, k2, tk3);
  const float dw1dn = ffma(c.pp, k1, -tk3);
  const float dw1dp = fmul(c.n, k1);
  const float dw1dq = ffma(-c.m, k1, sk3);
  const float dw2dp = ffma(c.n, k2, -sk3);
  const float dw2dn = fmul(c.pp, k2);
  const float dw2dq = -fmul(c.m, k2);
  const float n1ay = fadd(c.nk3n, fadd(dw1dp, dw1dq));
  const float n1ax = fadd(c.qk3, fadd(dw1dm, dw1dn));
  const float n2ax = fadd(c.ppk3n, fadd(dw2dm, dw2dn));
  const float n2ay = fadd(c.mk3, fadd(dw2dp, dw2dq));
#pragma unroll
  for (int d = 0; d < DT; ++d) {
    const float dl = fmul(g[d], c.rk);
    const float d1 = c.d1[d], d2 = c.d2[d];
    acc[0] = ffma(ffma(-n2ax, d2, -fmul(n1ax, d1)), dl, acc[0]);
    acc[1] = ffma(ffma(-n2ay, d2, -fmul(n1ay, d1)), dl, acc[1]);
    acc[2] = ffma(ffma(dw1dm, d1, fmul(dw2dm, d2)), dl, acc[2]);
    acc[3] = ffma(ffma(dw1dp, d1, fmul(dw2dp, d2)), dl, acc[3]);
    acc[4] = ffma(ffma(dw1dn, d1, fmul(dw2dn, d2)), dl, acc[4]);
    acc[5] = ffma(ffma(dw1dq, d1, fmul(dw2dq, d2)), dl, acc[5]);
    acc[6 + d] = ffma(g[d], aw, acc[6 + d]);
    acc[6 + DT + d] = ffma(g[d], bw, acc[6 + DT + d]);
    acc[6 + 2 * DT + d] = ffma(g[d], cw, acc[6 + 2 * DT + d]);
  }
}

#define DIBR_ROWS_MINB 16  /* H100 700 W, c4_shard, weights recomputed: 16 warps/SM 0.452 ms, 12: 0.453, 20: 0.455 */
template <int DT, typename FT>
__global__ void __launch_bounds__(32, DIBR_ROWS_MINB) raster_bwd_rows_kernel(const __grid_constant__ RowBwdArgs a) {
  using C = RwCfg<DT>;
  using G = RwG<DT, FT>;
  __shared__ __align__(128) unsigned char smem[2 * G::kStage];
  const int lane = threadIdx.x;
  // persistent single-warp CTAs pull (view, 32-row band, column strip) jobs from a counter: the
  // jobs differ by 10x in cost (background vs dense mesh), so a static grid ends with a
  // ragged tail of half-empty SMs
  const int total_jobs = a.jobs_x * a.jobs_y * a.B;
  for (;;) {
  int job = 0;
  if (lane == 0) job = atomicAdd(a.job_ctr, 1);
  job = __shfl_sync(kFull, job, 0);
  if (job >= total_jobs) break;
  const int jx = job % a.jobs_x; job /= a.jobs_x;
  const int jy = job % a.jobs_y;
  const int b = job / a.jobs_y;
  const int row0 = jy * 32, col0 = jx * a.strip;
  const int col1 = min(a.W, col0 + a.strip);
  const int nslabs = (col1 - col0) / kRwSlab;
  const bool row_ok = row0 + lane < a.H;
  const int64_t pix0 = ((int64_t)b * a.H + row0) * a.W;  // first pixel of the job's first row
  const int64_t fbase = (int64_t)b * a.F;
  const float y0 = pix_y(a.grid, row0 + lane);                            // the lane's row centre
  const float* wrow = a.w ? a.w + (pix0 + (int64_t)lane * a.W) * 3 : nullptr;   // given weights

  auto issue = [&](int s, int buf) {
    unsigned char* base = smem + buf * G::kStage;
    const int x = col0 + s * kRwSlab;
#pragma unroll
    for (int j = 0; j < 2; ++j) {           // face_idx: 2 chunks per row
      const int k = lane + 32 * j, r = k >> 1, ch = k & 1;
      if (row0 + r < a.H)
        cp_async16(base + r * C::kIdxPitch + ch * 16,
                   reinterpret_cast<const char*>(a.idx + pix0 + (int64_t)r * a.W + x) + ch * 16);
    }
    constexpr int GC = G::kRow / G::kChunk;   // upstream gradient: chunks per row
    const FT* gsrc = static_cast<const FT*>(a.grad_feat);
#pragma unroll
    for (int j = 0; j < GC; ++j) {
      const int k = lane + 32 * j, r = k / GC, ch = k - r * GC;
      if (row0 + r < a.H) {
        unsigned char* dst = base + 32 * C::kIdxPitch + r * G::kPitch + ch * G::kChunk;
        const char* src = reinterpret_cast<const char*>(gsrc + (pix0 + (int64_t)r * a.W + x) * DT) + ch * G::kChunk;
        if (G::kChunk == 16) cp_async16(dst, src); else cp_async8(dst, src);
      }
    }
    cp_async_commit();
  };

  int cur = -1;
  RowFace<DT> fc;
  float acc[C::kAcc];
#pragma unroll
  for (int i = 0; i < C::kAcc; ++i) acc[i] = 0.f;

  auto flush = [&]() {
    float4* p = reinterpret_cast<float4*>(a.acc + (fbase + cur) * C::kAcc);
#pragma unroll
    for (int i = 0; i < C::kAcc; i += 4) atomicAdd(p + (i >> 2), make_float4(acc[i], acc[i + 1], acc[i + 2], acc[i + 3]));
  };

  if (nslabs > 0) issue(0, 0);
  for (int s = 0; s < nslabs; ++s) {
    if (s + 1 < nslabs) { issue(s + 1, (s + 1) & 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
    __syncwarp();
    const unsigned char* base = smem + (s & 1) * G::kStage;
    if (row_ok) {
      do {
        const ulonglong2* ip = reinterpret_cast<const ulonglong2*>(base + lane * C::kIdxPitch);
        const ulonglong2 i01 = ip[0], i23 = ip[1];
        int f[4] = {(int)(long long)i01.x, (int)(long long)i01.y, (int)(long long)i23.x, (int)(long long)i23.y};
        bool any = cur >= 0;
#pragma unroll
        for (int p = 0; p < 4; ++p) { f[p] = f[p] < 0 ? -1 : f[p]; any = any || f[p] >= 0; }
        if (!any) break;
        float gv[4 * DT];
        {
          const unsigned char* grow = base + 32 * C::kIdxPitch + lane * G::kPitch;
          if (std::is_same<FT, float>::value) {
            const float4* gp = reinterpret_cast<const float4*>(grow);
#pragma unroll
            for (int k = 0; k < DT; ++k) { const float4 t = gp[k]; gv[4 * k] = t.x; gv[4 * k + 1] = t.y; gv[4 * k + 2] = t.z; gv[4 * k + 3] = t.w; }
          } else {   // bf16: 2 values per 32-bit word, low half first
            const uint2* gp = reinterpret_cast<const uint2*>(grow);
#pragma unroll
            for (int k = 0; k < DT; ++k) {
              const uint2 t = gp[k];
              gv[4 * k] = __uint_as_float(t.x << 16); gv[4 * k + 1] = __uint_as_float(t.x & 0xffff0000u);
              gv[4 * k + 2] = __uint_as_float(t.y << 16); gv[4 * k + 3] = __uint_as_float(t.y & 0xffff0000u);
            }
          }
        }
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          if (f[p] != cur) {
            if (cur >= 0) flush();
            cur = f[p];
            if (cur >= 0) {
              row_face_load<DT, FT>(a, fbase + cur, fc);
#pragma unroll
              for (int i = 0; i < C::kAcc; ++i) acc[i] = 0.f;
            }
          }
          if (cur >= 0) {
            const int x = col0 + s * kRwSlab + p;
            float aw, bw, cw;
            if (wrow) {
              aw = __ldcs(wrow + 3 * x); bw = __ldcs(wrow + 3 * x + 1); cw = __ldcs(wrow + 3 * x + 2);
            } else {
              raster_weights_of(a.rc, pix_x(a.grid, x), y0, fc.mx[0], fc.my[0], fc.mx[1], fc.my[1],
                                fc.mx[2], fc.my[2], aw, bw, cw);
            }
            row_pixel<DT>(fc, aw, bw, cw, &gv[DT * p], acc);
          }
        }
      } while (false);
    }
    __syncwarp();  // everyone is done with this buffer before slab s+2 lands in it
  }
  if (cur >= 0) flush();
  __syncwarp();
  }  // job loop
}

// acc[face][kAcc] -> grad_face_vertices_image (NF,3,2) (= or +=) and grad_face_features (NF,3,D) (=).
// A CTA moves 256 face records through shared memory so that both the 64-byte records and the
// 24- / 12*D-byte output rows are read and written as contiguous, fully used lines.
template <int DT>
__global__ void __launch_bounds__(256) raster_bwd_finalize_kernel(const float* __restrict__ acc, int64_t NF,
                                                                 float* __restrict__ g_xy, float* __restrict__ g_ff,
                                                                 int accumulate_xy) {
  using C = RwCfg<DT>;
  constexpr int kFaces = 256;
  __shared__ __align__(16) float sm[kFaces * C::kAcc];
  const int64_t f0 = (int64_t)blockIdx.x * kFaces;
  const int nf = (int)min((int64_t)kFaces, NF - f0);
  const int tid = threadIdx.x;
  const float4* src = reinterpret_cast<const float4*>(acc + f0 * C::kAcc);
  for (int i = tid; i < nf * (C::kAcc / 4); i += 256) reinterpret_cast<float4*>(sm)[i] = __ldcs(src + i);
  __syncthreads();
  float2* gx = reinterpret_cast<float2*>(g_xy + f0 * 6);
  for (int i = tid; i < nf * 3; i += 256) {          // (face, vertex) -> float2
    const int f = i / 3, v = i - f * 3;
    float2 o = make_float2(sm[f * C::kAcc + 2 * v], sm[f * C::kAcc + 2 * v + 1]);
    if (accumulate_xy) { const float2 p = gx[i]; o.x += p.x; o.y += p.y; }
    gx[i] = o;
  }
  float* gf = g_ff + f0 * 3 * DT;
  for (int i = tid; i < nf * 3 * DT; i += 256) {
    const int f = i / (3 * DT), j = i - f * (3 * DT);
    gf[i] = sm[f * C::kAcc + 6 + j];
  }
}

// ---------------------------------------------------------------------------
// Soft-mask backward from stored K-lists (operator contract, dibr_soft_mask_cuda.cu:230-353).
struct SoftBwdListArgs {
  int B, H, W, F, K;
  PixelGrid grid;
  float sigmainv, multiplier;
  const float* grad_soft; const float* soft; const int64_t* idx;
  const float* prob; const int64_t* cidx; const uint8_t* ctype; const float* xy;
  float* grad_xy;
};

__global__ void __launch_bounds__(256) soft_bwd_lists_kernel(const __grid_constant__ SoftBwdListArgs a) {
  const int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t P = (int64_t)a.B * a.H * a.W;
  if (pix >= P) return;
  if (a.idx[pix] >= 0) return;
  const int ix = (int)(pix % a.W);
  const int iy = (int)((pix / a.W) % a.H);
  const int64_t b = pix / ((int64_t)a.W * a.H);
  const float x0 = pix_x(a.grid, ix), y0 = pix_y(a.grid, iy);
  const float dLdp = a.grad_soft[pix], allprob = a.soft[pix];
  for (int k = 0; k < a.K; ++k) {
    const int64_t f = a.cidx[pix * a.K + k];
    if (f < 0) break;
    const int64_t base = (b * a.F + f) * 6;
    float v[6], g[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) v[i] = __ldg(a.xy + base + i);
    soft_backward_terms(x0, y0, v, (int)a.ctype[pix * a.K + k] - 1, a.prob[pix * a.K + k], allprob,
                        dLdp, a.sigmainv, a.multiplier, g);
#pragma unroll
    for (int i = 0; i < 6; ++i)
      if (g[i] != 0.f) atomicAdd(a.grad_xy + base + i, g[i]);
  }
}

// ---------------------------------------------------------------------------
// Host side.
int check_dims(int B, int64_t NF, int H, int W) {
  if (B <= 0 || H <= 0 || W <= 0 || NF < 0) return DIBR_B200_EINVAL;
  if (H > DIBR_B200_MAX_IMAGE_DIM || W > DIBR_B200_MAX_IMAGE_DIM || B > 65535) return DIBR_B200_ESIZE;
  if (NF > 0x3fffffffLL) return DIBR_B200_ESIZE;
  return 0;
}

// Carves the scene's pieces out of the workspace (workspace_layout.h).  knum > 0 enables the hit
// cache in whatever the workspace holds beyond the minimum; f64 adds the float scene of a float64
// call, which f64_bins fills in.  The other face inputs (xy, z, first, validity, given bboxes) are
// left empty for the caller to fill in.
int setup_scene(Scene& s, int B, int64_t NF, int F, int H, int W, float multiplier, float margin,
                int knum, bool f64, void* ws, size_t ws_bytes) {
  if (!(multiplier > 0.f)) return DIBR_B200_EINVAL;
  if (!ws) return DIBR_B200_EINVAL;
  const WorkspaceLayout L = workspace_layout({B, NF, H, W, knum, f64}, ws, ws_bytes);
  if (!L.fits) return DIBR_B200_EWORKSPACE;
  char* const o = (char*)ws + L.origin;
  s.first = nullptr; s.xy = nullptr; s.z = nullptr; s.premultiplied = 0;
  s.fnz = nullptr; s.valid = nullptr; s.bbox_tight = nullptr; s.bbox_large = nullptr;
  s.B = B; s.H = H; s.W = W; s.F = F; s.NF = NF;
  s.multiplier = multiplier; s.margin = margin;
  s.grid = make_grid(multiplier, W, H);
  s.L = levels_for(H, W);
  int nb = 0;
  for (int l = 0; l < kMaxLevels; ++l) {
    const int t = kTile << (2 * l);
    s.ntx[l] = l < s.L ? (W + t - 1) / t : 0;
    s.nty[l] = l < s.L ? (H + t - 1) / t : 0;
    s.bin_base[l] = nb;
    nb += s.ntx[l] * s.nty[l];
  }
  s.NB = nb;
  if ((int64_t)2 * B * nb >= 0x7fffffffLL) return DIBR_B200_ESIZE;  // counter ids are 32-bit
  s.cnt = (int*)(o + L.cnt.at);
  s.pool_ctr = (int*)(o + L.pool_ctr.at);
  s.fb_ctr = (int*)(o + L.fb_ctr.at);
  s.band_ctr = (int*)(o + L.band_ctr.at);
  s.view_flag = (int*)(o + L.view_flag.at);
  s.tile_cnt = (int*)(o + L.tile_cnt.at);
  s.off = (int*)(o + L.off.at);
  s.fb_list = (int*)(o + L.fb_list.at);
  s.band_list = (int*)(o + L.band_list.at);
  s.entries = (int4*)(o + L.entries.at);
  s.pool_tiles = (int)L.cache_tiles; s.pool_K = knum > 0 ? knum : 1;
  s.pool_hdr = L.cache_tiles ? (int4*)(o + L.cache_hdr.at) : nullptr;
  s.pool_data = L.cache_tiles ? (uint32_t*)(o + L.cache_data.at) : nullptr;
  if (f64) {
    s.xy = (float*)(o + L.xy.at); s.premultiplied = 1;
    s.bbox_tight = (float*)(o + L.bbox_tight.at);
    s.bbox_large = (float*)(o + L.bbox_large.at);
    s.valid = (uint8_t*)(o + L.valid.at);
  }
  return 0;
}

int build_bins(const Scene& s, int sets, cudaStream_t st) {
  const Piece counters = workspace_layout({s.B, s.NF, s.H, s.W, 0, false}, 0).counters;
  cudaError_t e = cudaMemsetAsync(s.cnt, 0, counters.bytes, st);
  if (e != cudaSuccess) return (int)e;
  if (s.NF > 0) {
    // dense meshes (tens of faces per 16x16 tile) hammer a few counters: aggregate per CTA.  Sparse
    // meshes of equal-sized views whose counters (and bitmask words) fit kBinChunkSmemBudget count and
    // fill in view-owned chunks (c2, c3, c4_shard); the others (large images, packed batches, whose
    // view sizes the host does not know) take plain atomics.
    const bool agg = s.NF / s.B >= (int64_t)32 * s.ntx[0] * s.nty[0];
    const size_t chunk_smem = (size_t)bin_chunk_words(s, sets) * sizeof(int);
    const bool chunked = !agg && !s.first && chunk_smem <= kBinChunkSmemBudget;
    const int threads = agg ? kBinThreadsAgg : kBinThreadsPlain;
    const unsigned blocks = (unsigned)((s.NF + threads - 1) / threads);
    {
      Span sp("bin_faces_kernel<count>", st);
      if (chunked) {
        // chunks of 256..2048 faces (1..8 per thread), as large as still gives kBinChunkTargetCtas CTAs
        int64_t per_thread = s.NF / ((int64_t)kBinChunkTargetCtas * kBinChunkThreads);
        per_thread = per_thread < 1 ? 1 : per_thread > kBinChunkMaxPerThread ? kBinChunkMaxPerThread : per_thread;
        const int chunk = kBinChunkThreads * (int)per_thread;
        const dim3 grid((unsigned)((s.F + chunk - 1) / chunk), (unsigned)s.B);
        bin_count_chunk_kernel<<<grid, kBinChunkThreads, chunk_smem, st>>>(s, sets, chunk);
      } else if (agg) {
        bin_faces_kernel<false, true><<<blocks, threads, 0, st>>>(s, sets);
      } else {
        bin_faces_kernel<false, false><<<blocks, threads, 0, st>>>(s, sets);
      }
    }
    {
      Span sp("scan_bins_kernel", st);
      scan_bins_kernel<<<2 * s.B, 1024, 0, st>>>(s);
    }
    {
      Span sp("bin_faces_kernel<fill>", st);
      if (chunked) {
        const dim3 grid((unsigned)((s.F + kBinChunkThreads - 1) / kBinChunkThreads), (unsigned)s.B);
        const size_t fill_smem = (size_t)((sets & 1) + ((sets >> 1) & 1)) * s.NB * sizeof(int);
        bin_fill_chunk_kernel<<<grid, kBinChunkThreads, fill_smem, st>>>(s, sets);
      } else if (agg) bin_faces_kernel<true, true><<<blocks, threads, 0, st>>>(s, sets);
      else bin_faces_kernel<true, false><<<blocks, threads, 0, st>>>(s, sets);
    }
  }
  return (int)cudaGetLastError();
}

dim3 tile_grid(const Scene& s) { return dim3((unsigned)s.ntx[0], (unsigned)s.nty[0], (unsigned)s.B); }

// CTAs of `kernel` resident on the current device at `threads` threads and `dyn_smem` bytes of
// dynamic shared memory (SMs x CTAs per SM; `per_sm_guess` per SM if the query fails), for the
// persistent kernels.  A property of (device, kernel): queried once and cached in a table
// (idempotent writes of the same value, safe from any thread) - the occupancy / attribute
// queries add host time to every call when repeated.
struct WaveEntry { const void* kernel; int dev; int wave; };
constexpr int kWaveSlots = 256;   // 12 persistent instantiations per device
WaveEntry g_waves[kWaveSlots];    // append-only; a lost race re-queries and stores the same value again

template <typename Kernel>
int resident_ctas(Kernel kernel, int threads, int per_sm_guess, size_t dyn_smem = 0) {
  int dev = 0;
  cudaGetDevice(&dev);
  const void* key = reinterpret_cast<const void*>(kernel);   // kernels with one signature share this template
  for (int i = 0; i < kWaveSlots && g_waves[i].kernel; ++i)
    if (g_waves[i].kernel == key && g_waves[i].dev == dev) return g_waves[i].wave;
  int sms = 132, per_sm = per_sm_guess;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (dyn_smem > 48 * 1024)
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_smem);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, dyn_smem) != cudaSuccess || per_sm < 1)
    per_sm = per_sm_guess;
  const int wave = sms * per_sm;
  for (int i = 0; i < kWaveSlots; ++i)
    if (!g_waves[i].kernel) { g_waves[i].dev = dev; g_waves[i].wave = wave; g_waves[i].kernel = key; break; }
  return wave;
}

// Persistent tile kernels: one resident wave, never more than the tiles.
template <typename Kernel>
unsigned persistent_grid(const Scene& s, Kernel kernel, size_t dyn_smem = 0) {
  const int wave = resident_ctas(kernel, kThreads, 2, dyn_smem);
  const int64_t ntiles = (int64_t)s.ntx[0] * s.nty[0] * s.B;
  return (unsigned)(ntiles < wave ? ntiles : wave);
}

template <bool R, bool S, bool K, typename FT = float>
void launch_fwd(const FwdArgs& a0, cudaStream_t st) {
  static_assert(!(R && K), "the K-lists come from the soft-mask-only forward");
  FwdArgs a = a0;
  a.from_fb = 0;
  {
    // dibr_fwd2_kernel (32x32 px per CTA, candidates staged once for 4 tiles) when the mesh is
    // sparse enough for a 32x32 tile's candidates to fit one staging round and the grid still
    // fills the GPU; dense meshes / small images keep one tile per CTA.
    const int64_t tiles32 = (int64_t)((a.s.W + 31) / 32) * ((a.s.H + 31) / 32);
    const int64_t faces_per_view = a.s.NF / (a.s.B > 0 ? a.s.B : 1);
    // ~ faces per 32x32 tile <= 40: c4 (20 k faces at 1024^2) has 20, c3 (512^2) 80, c2 80, c5 320
    const bool two = R && faces_per_view <= 40 * tiles32 && tiles32 * a.s.B >= 2048;
    if (two) {
      Span sp("dibr_fwd2_kernel<S=2>", st);
      const dim3 grid((unsigned)((a.s.ntx[0] + 1) / 2), (unsigned)((a.s.nty[0] + 1) / 2), (unsigned)a.s.B);
      if constexpr (R) dibr_fwd2_kernel<S, FT><<<grid, kThreads, 0, st>>>(a);
    } else {
      // one 16x16 tile per CTA: dense meshes (hundreds of candidates per tile) and small images
      Span sp("dibr_tile_fwd_kernel", st);
      dibr_tile_fwd_kernel<R, S, K, FT><<<tile_grid(a.s), kThreads, 0, st>>>(a);
    }
  }
  if (S) {
    const unsigned g1 = persistent_grid(a.s, soft_tiles_fwd_kernel<K>, sizeof(SoftSmem));   // (sets the smem attribute once)
    if (!K && a.cache && a.s.pool_tiles > 0 && a.K <= kSoftFwdK) {
      // enumerate, evaluate densely and fold per tile; tiles beyond the cache take the single-kernel path
      {
        Span sp("soft_fwd_kernel", st);
        soft_fwd_kernel<<<persistent_grid(a.s, soft_fwd_kernel), kThreads, 0, st>>>(a);
      }
      a.from_fb = 1;
      a.cache = 0;
      Span sp("soft_tiles_fwd_kernel<leftovers>", st);
      soft_tiles_fwd_kernel<K><<<g1, kThreads, sizeof(SoftSmem), st>>>(a);
    } else {
      Span sp("soft_tiles_fwd_kernel", st);
      soft_tiles_fwd_kernel<K><<<g1, kThreads, sizeof(SoftSmem), st>>>(a);
    }
  }
}

template <typename FT>
int launch_raster_bwd(const RasterBwdArgs& a, cudaStream_t st) {
  const dim3 grid((unsigned)a.ntx, (unsigned)a.nty, (unsigned)a.B);
  Span sp("raster_bwd_kernel", st);
  switch (a.D) {
    case 1: raster_bwd_kernel<1, FT><<<grid, kThreads, 0, st>>>(a); break;
    case 2: raster_bwd_kernel<2, FT><<<grid, kThreads, 0, st>>>(a); break;
    case 3: raster_bwd_kernel<3, FT><<<grid, kThreads, 0, st>>>(a); break;
    case 4: raster_bwd_kernel<4, FT><<<grid, kThreads, 0, st>>>(a); break;
    default: raster_bwd_kernel<0, FT><<<grid, kThreads, 0, st>>>(a); break;
  }
  return (int)cudaGetLastError();
}

template <int DT, typename FT>
int launch_rows_t(const RowBwdArgs& a, int64_t NF, float* g_xy, float* g_ff, int accumulate_xy, cudaStream_t st) {
  // the face records and the job counter right behind them
  cudaError_t e = cudaMemsetAsync(a.acc, 0, (size_t)((char*)(a.job_ctr + 1) - (char*)a.acc), st);
  if (e != cudaSuccess) return (int)e;
  {
    Span sp("raster_bwd_rows_kernel", st);
    const int slots = resident_ctas(raster_bwd_rows_kernel<DT, FT>, 32, DIBR_ROWS_MINB);
    const int64_t jobs = (int64_t)a.jobs_x * a.jobs_y * a.B;
    raster_bwd_rows_kernel<DT, FT><<<(unsigned)(jobs < slots ? jobs : slots), 32, 0, st>>>(a);
  }
  {
    Span sp("raster_bwd_finalize_kernel", st);
    raster_bwd_finalize_kernel<DT><<<(unsigned)((NF + 255) / 256), 256, 0, st>>>(a.acc, NF, g_xy, g_ff, accumulate_xy);
  }
  return (int)cudaGetLastError();
}

// Row-walk rasterize backward: one warp per 32 rows x strip columns; the strip is as long as
// still leaves a few waves of single-warp CTAs (longer strips = fewer cut face runs).
template <typename FT>
int launch_raster_bwd_rows(const RasterBwdArgs& r, float* acc, int* job_ctr, int accumulate_xy, cudaStream_t st) {
  RowBwdArgs a;
  a.B = r.B; a.H = r.H; a.W = r.W; a.F = r.F;
  a.grad_feat = r.grad_feat; a.idx = r.idx; a.w = r.w; a.xy = r.xy;
  a.feat = r.feat; a.grid = r.grid; a.rc = r.rc; a.multiplier = r.multiplier;
  a.acc = acc; a.job_ctr = job_ctr;
  a.jobs_y = (r.H + 31) / 32;
  int strip = 32;   // H100, c4_shard: strips of 16 / 64 columns 1 % faster / 8 % slower
  while (strip > kRwSlab && (int64_t)r.B * a.jobs_y * ((r.W + strip - 1) / strip) < 8192) strip >>= 1;
  a.strip = strip;
  a.jobs_x = (r.W + strip - 1) / strip;
  const int64_t NF = (int64_t)r.B * r.F;
  switch (r.D) {
    case 1: return launch_rows_t<1, FT>(a, NF, r.grad_xy, r.grad_feat_out, accumulate_xy, st);
    case 2: return launch_rows_t<2, FT>(a, NF, r.grad_xy, r.grad_feat_out, accumulate_xy, st);
    case 3: return launch_rows_t<3, FT>(a, NF, r.grad_xy, r.grad_feat_out, accumulate_xy, st);
    case 4: return launch_rows_t<4, FT>(a, NF, r.grad_xy, r.grad_feat_out, accumulate_xy, st);
    default: return DIBR_B200_EINVAL;
  }
}

#include "dibr_f64.cuh"

// Whether every non-null tensor pointer starts on a 16-byte boundary.  The kernels read and write
// the caller's tensors with float2 / float4 / int4 accesses and 16-byte cp.async copies at offsets
// that are multiples of the vector size from the tensor's start, so only the start is checked.
bool aligned16(std::initializer_list<const void*> ptrs) {
  for (const void* p : ptrs)
    if (reinterpret_cast<uintptr_t>(p) & 15) return false;
  return true;
}

// The argument checks of the fused forward (dibr_b200_forward, _bf16, _f64).  The float32/bf16
// forward may leave output_weights NULL (nothing is written there then); the float64 one stores them.
int check_forward(bool f64, int B, int F, int H, int W, int D, int mode, const void* fvz, const void* fvi,
                  const void* ff, const void* fnz, const void* valid, float multiplier, int knum,
                  const void* out_feat, const int64_t* face_idx, const void* out_w, const void* soft_mask) {
  const int rc = check_dims(B, (int64_t)B * F, H, W);
  if (rc) return rc;
  if (!aligned16({fvz, fvi, ff, fnz, valid, out_feat, face_idx, out_w, soft_mask})) return DIBR_B200_EINVAL;
  const bool raster = mode & DIBR_B200_RASTER, soft = mode & DIBR_B200_SOFT_MASK;
  if ((!raster && !soft) || F < 0 || D < 0 || !face_idx || (f64 && !(multiplier > 0.f))) return DIBR_B200_EINVAL;
  if (F > 0 && !fvi) return DIBR_B200_EINVAL;
  if (raster && ((f64 && !out_w) || (D > 0 && (!out_feat || (F > 0 && !ff))) || (F > 0 && !fvz)))
    return DIBR_B200_EINVAL;
  if (soft && (!soft_mask || knum <= 0)) return DIBR_B200_EINVAL;
  return 0;
}

// The argument checks of the fused backward (dibr_b200_backward, _bf16, _views, _f64), all of them
// made before anything is enqueued: a call that fails them writes no output.  On success `s` holds
// the scene of the branches that need one (float32/bf16: the soft-mask branch; float64: either).
int check_backward(bool f64, int B, int F, int H, int W, int D, const void* grad_features,
                   const void* grad_soft_mask, const int64_t* face_idx, const void* output_weights,
                   const void* soft_mask, const void* fvi, const void* ff, float multiplier, float boxlen_m,
                   int knum, const void* g_fvi, const void* g_ff, void* ws, size_t ws_bytes, int view_begin,
                   int view_end, Scene& s) {
  const int64_t NF = (int64_t)B * F;
  const int rc = check_dims(B, NF, H, W);
  if (rc) return rc;
  if (!aligned16({grad_features, grad_soft_mask, face_idx, output_weights, soft_mask, fvi, ff, g_fvi, g_ff}))
    return DIBR_B200_EINVAL;
  if (!face_idx || !g_fvi || F < 0 || D < 0 || (f64 && !(multiplier > 0.f))) return DIBR_B200_EINVAL;
  if (F > 0 && !fvi) return DIBR_B200_EINVAL;
  if (view_begin < 0 || view_end > B || view_begin >= view_end) return DIBR_B200_EINVAL;
  const bool raster = grad_features && D > 0;
  const bool soft_ok = !grad_soft_mask || (soft_mask && knum > 0);
  if (f64 && !soft_ok) return DIBR_B200_EINVAL;     // the float64 backward refuses it even without faces
  if (NF == 0) return 0;                            // no faces: the gradients are only zeroed
  // without stored weights the float32/bf16 rasterize branch recomputes them with the multiplier
  if (raster && (!ff || !g_ff || !(output_weights || (!f64 && multiplier > 0.f)))) return DIBR_B200_EINVAL;
  if (!soft_ok) return DIBR_B200_EINVAL;
  if (f64) return raster || grad_soft_mask ? f64_scene(s, B, F, H, W, multiplier, ws, ws_bytes) : 0;
  return grad_soft_mask ? setup_scene(s, B, NF, F, H, W, multiplier, boxlen_m, knum, false, ws, ws_bytes) : 0;
}

}  // namespace

// The launch trace for the library's other sources (mesh_topology.cu): the same events as Span.
namespace dibr_b200_detail {
bool span_open(const char* name, cudaStream_t st) {
  Span s(name, st);        // records the opening event when a trace is open
  const bool on = s.on;
  s.on = false;            // span_close records the closing one
  return on;
}
void span_close(cudaStream_t st) {
  cudaEventRecord(g_trace.pool[g_trace.used + 1], st);
  g_trace.used += 2;
}
}  // namespace dibr_b200_detail

// ===========================================================================
extern "C" {

size_t dibr_b200_workspace_bytes_f64(int batch, int64_t total_faces, int height, int width) {
  if (check_dims(batch, total_faces, height, width)) return 0;
  return workspace_layout({batch, total_faces, height, width, 0, true}, 0).bytes;
}

int dibr_b200_forward_f64(int batch, int num_faces, int height, int width, int feat_dim,
                          const double* face_vertices_z, const double* face_vertices_image,
                          const double* face_features, const double* face_normals_z, const uint8_t* valid_faces,
                          double multiplier, float eps, int mode, float sigmainv, double boxlen_m, int knum,
                          double* interpolated_features, int64_t* face_idx, double* output_weights,
                          double* soft_mask, void* workspace, size_t workspace_bytes_, dibr_b200_stream_t stream) {
  const float multiplier_f = (float)multiplier;      // the reference kernels' float parameter
  int rc = check_forward(true, batch, num_faces, height, width, feat_dim, mode, face_vertices_z, face_vertices_image,
                         face_features, face_normals_z, valid_faces, multiplier_f, knum, interpolated_features, face_idx,
                         output_weights, soft_mask);
  if (rc) return rc;
  const bool raster = mode & DIBR_B200_RASTER, soft = mode & DIBR_B200_SOFT_MASK;
  cudaStream_t st = (cudaStream_t)stream;
  F64Args a;
  rc = f64_scene(a.s, batch, num_faces, height, width, multiplier_f, workspace, workspace_bytes_);
  if (rc) return rc;
  rc = f64_bins(a.s, face_vertices_image, face_vertices_z, face_normals_z, valid_faces, multiplier, boxlen_m,
                (raster ? 1 : 0) | (soft ? 2 : 0), st);
  if (rc) return rc;
  a.D = feat_dim; a.K = knum; a.mode = mode; a.eps = eps; a.sigmainv = sigmainv; a.multiplier = multiplier_f;
  a.scale = multiplier;
  a.margin = boxlen_m; a.xy = face_vertices_image; a.z = face_vertices_z; a.feat = face_features;
  a.out_feat = interpolated_features; a.idx = face_idx; a.out_w = output_weights; a.out_soft = soft_mask;
  a.g_feat = nullptr; a.g_soft = nullptr; a.soft = nullptr; a.g_xy = nullptr; a.g_ff = nullptr;
  Span sp("dibr_f64_kernel<forward>", st);
  dibr_f64_kernel<false><<<tile_grid(a.s), kThreads, 0, st>>>(a);
  return (int)cudaGetLastError();
}

int dibr_b200_backward_f64(int batch, int num_faces, int height, int width, int feat_dim,
                           const double* grad_features, const double* grad_soft_mask, const int64_t* face_idx,
                           const double* output_weights, const double* soft_mask, const double* face_vertices_image,
                           const double* face_features, double multiplier, float eps, float sigmainv, double boxlen_m,
                           int knum, double* grad_face_vertices_image, double* grad_face_features, void* workspace,
                           size_t workspace_bytes_, int flags, dibr_b200_stream_t stream) {
  const int64_t NF = (int64_t)batch * num_faces;
  const float multiplier_f = (float)multiplier;      // the reference kernels' float parameter
  F64Args a;
  int rc = check_backward(true, batch, num_faces, height, width, feat_dim, grad_features, grad_soft_mask, face_idx,
                          output_weights, soft_mask, face_vertices_image, face_features, multiplier_f, 0.f, knum,
                          grad_face_vertices_image, grad_face_features, workspace, workspace_bytes_, 0, batch, a.s);
  if (rc) return rc;
  const bool run_raster = grad_features && feat_dim > 0;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(grad_face_vertices_image, 0, (size_t)NF * 6 * sizeof(double), st);
  if (e != cudaSuccess) return (int)e;
  if (grad_face_features && feat_dim > 0) {
    e = cudaMemsetAsync(grad_face_features, 0, (size_t)NF * 3 * feat_dim * sizeof(double), st);
    if (e != cudaSuccess) return (int)e;
  }
  if (NF == 0 || (!run_raster && !grad_soft_mask)) return 0;
  // the soft-mask branch needs the enlarged bins: forward's (BINS_VALID) or rebuilt here
  if (grad_soft_mask && !(flags & DIBR_B200_BINS_VALID)) {
    rc = f64_bins(a.s, face_vertices_image, nullptr, nullptr, nullptr, multiplier, boxlen_m, 2, st);
    if (rc) return rc;
  }
  a.D = feat_dim; a.K = knum; a.mode = 0; a.eps = eps; a.sigmainv = sigmainv; a.multiplier = multiplier_f;
  a.scale = multiplier;
  a.margin = boxlen_m; a.xy = face_vertices_image; a.z = nullptr; a.feat = face_features;
  a.out_feat = nullptr; a.idx = const_cast<int64_t*>(face_idx); a.out_w = const_cast<double*>(output_weights);
  a.out_soft = nullptr; a.g_feat = run_raster ? grad_features : nullptr; a.g_soft = grad_soft_mask; a.soft = soft_mask;
  a.g_xy = grad_face_vertices_image; a.g_ff = grad_face_features;
  Span sp("dibr_f64_kernel<backward>", st);
  dibr_f64_kernel<true><<<tile_grid(a.s), kThreads, 0, st>>>(a);
  return (int)cudaGetLastError();
}

int dibr_b200_trace_begin(void) {
  g_trace.on = true;
  g_trace.used = 0;
  g_trace.names.clear();
  return 0;
}

int dibr_b200_trace_end(char* names, size_t names_bytes, float* ms, int capacity) {
  TraceState& t = g_trace;
  t.on = false;
  const int n = t.used / 2;
  std::string joined;
  for (int i = 0; i < n; ++i) {
    if (cudaEventSynchronize(t.pool[2 * i + 1]) != cudaSuccess) return DIBR_B200_EINVAL;
    float v = 0.f;
    if (cudaEventElapsedTime(&v, t.pool[2 * i], t.pool[2 * i + 1]) != cudaSuccess) return DIBR_B200_EINVAL;
    if (ms && i < capacity) ms[i] = v;
    joined += t.names[i];
    joined += '\n';
  }
  if (names && names_bytes > 0) {
    const size_t c = joined.size() < names_bytes - 1 ? joined.size() : names_bytes - 1;
    memcpy(names, joined.data(), c);
    names[c] = 0;
  }
  t.used = 0;
  t.names.clear();
  return n;
}

int dibr_b200_version(void) { return 200; }

size_t dibr_b200_workspace_bytes(int batch, int64_t total_faces, int height, int width) {
  if (check_dims(batch, total_faces, height, width)) return 0;
  return workspace_layout({batch, total_faces, height, width, 0, false}, 0).bytes;
}

size_t dibr_b200_workspace_bytes_cached(int batch, int64_t total_faces, int height, int width,
                                        int knum, int64_t cache_tiles) {
  if (check_dims(batch, total_faces, height, width) || knum <= 0 || cache_tiles < 0) return 0;
  return workspace_layout({batch, total_faces, height, width, knum, false}, cache_tiles).bytes;
}

static int forward_impl(int batch, int num_faces, int height, int width, int feat_dim,
                        const float* face_vertices_z, const float* face_vertices_image,
                        const void* face_features, const float* face_normals_z,
                        const uint8_t* valid_faces, float multiplier, float eps, int mode,
                        float sigmainv, float boxlen_m, int knum, void* interpolated_features,
                        int64_t* face_idx, float* output_weights, float* soft_mask, void* workspace,
                        size_t workspace_bytes_, dibr_b200_stream_t stream, bool bf16) {
  const int64_t NF = (int64_t)batch * num_faces;
  int rc = check_forward(false, batch, num_faces, height, width, feat_dim, mode, face_vertices_z, face_vertices_image,
                         face_features, face_normals_z, valid_faces, multiplier, knum, interpolated_features, face_idx,
                         output_weights, soft_mask);
  if (rc) return rc;
  const bool raster = mode & DIBR_B200_RASTER, soft = mode & DIBR_B200_SOFT_MASK;
  cudaStream_t st = (cudaStream_t)stream;
  FwdArgs a;
  Scene& s = a.s;
  rc = setup_scene(s, batch, NF, num_faces, height, width, multiplier, boxlen_m, soft ? knum : 0, false,
                   workspace, workspace_bytes_);
  if (rc) return rc;
  s.xy = face_vertices_image; s.z = face_vertices_z; s.fnz = face_normals_z; s.valid = valid_faces;
  rc = build_bins(s, (raster ? 1 : 0) | (soft ? 2 : 0), st);
  if (rc) return rc;
  a.rc = make_raster_const(eps);
  a.D = feat_dim; a.feat = face_features; a.sigmainv = sigmainv; a.K = knum;
  a.cache = soft ? 1 : 0;   // hits are cached while blocks last; other tiles go to fb_list
  a.out_feat = interpolated_features; a.idx = face_idx; a.out_w = output_weights; a.out_soft = soft_mask;
  a.kl = SoftFwdOut{nullptr, nullptr, nullptr};
  if (raster && soft) { if (bf16) launch_fwd<true, true, false, __nv_bfloat16>(a, st); else launch_fwd<true, true, false>(a, st); }
  else if (raster) { if (bf16) launch_fwd<true, false, false, __nv_bfloat16>(a, st); else launch_fwd<true, false, false>(a, st); }
  else launch_fwd<false, true, false>(a, st);
  return (int)cudaGetLastError();
}

int dibr_b200_forward(int batch, int num_faces, int height, int width, int feat_dim,
                      const float* face_vertices_z, const float* face_vertices_image,
                      const float* face_features, const float* face_normals_z,
                      const uint8_t* valid_faces, float multiplier, float eps, int mode,
                      float sigmainv, float boxlen_m, int knum, float* interpolated_features,
                      int64_t* face_idx, float* output_weights, float* soft_mask, void* workspace,
                      size_t workspace_bytes_, dibr_b200_stream_t stream) {
  return forward_impl(batch, num_faces, height, width, feat_dim, face_vertices_z, face_vertices_image,
                      face_features, face_normals_z, valid_faces, multiplier, eps, mode, sigmainv, boxlen_m,
                      knum, interpolated_features, face_idx, output_weights, soft_mask, workspace,
                      workspace_bytes_, stream, false);
}

int dibr_b200_forward_bf16(int batch, int num_faces, int height, int width, int feat_dim,
                           const float* face_vertices_z, const float* face_vertices_image,
                           const uint16_t* face_features, const float* face_normals_z,
                           const uint8_t* valid_faces, float multiplier, float eps, int mode,
                           float sigmainv, float boxlen_m, int knum, uint16_t* interpolated_features,
                           int64_t* face_idx, float* output_weights, float* soft_mask, void* workspace,
                           size_t workspace_bytes_, dibr_b200_stream_t stream) {
  return forward_impl(batch, num_faces, height, width, feat_dim, face_vertices_z, face_vertices_image,
                      face_features, face_normals_z, valid_faces, multiplier, eps, mode, sigmainv, boxlen_m,
                      knum, interpolated_features, face_idx, output_weights, soft_mask, workspace,
                      workspace_bytes_, stream, true);
}


static int backward_impl(int batch, int num_faces, int height, int width, int feat_dim,
                         const void* grad_features, const float* grad_soft_mask,
                         const int64_t* face_idx, const float* output_weights, const float* soft_mask,
                         const float* face_vertices_image, const void* face_features,
                         float multiplier, float eps, float sigmainv, float boxlen_m, int knum,
                         float* grad_face_vertices_image, float* grad_face_features, void* workspace,
                         size_t workspace_bytes_, int flags, dibr_b200_stream_t stream, bool bf16,
                         int view_begin, int view_end) {
  const int64_t NF = (int64_t)batch * num_faces;
  const bool bins_valid = (flags & DIBR_B200_BINS_VALID) != 0;
  SoftBwdArgs sa;   // the soft-mask branch's arguments: check_backward sets up its scene
  int rc = check_backward(false, batch, num_faces, height, width, feat_dim, grad_features, grad_soft_mask, face_idx,
                          output_weights, soft_mask, face_vertices_image, face_features, multiplier, boxlen_m, knum,
                          grad_face_vertices_image, grad_face_features, workspace, workspace_bytes_, view_begin,
                          view_end, sa.s);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaSuccess;
  const bool run_raster = grad_features && feat_dim > 0;
  // the views of this call: rows [view_begin, view_end) of every per-view tensor
  const int nv = view_end - view_begin;
  const int64_t NFv = (int64_t)nv * num_faces;
  const size_t fsz = bf16 ? 2 : 4;
  float* const g_xy_v = grad_face_vertices_image + (size_t)view_begin * num_faces * 6;
  float* const g_ff_v = grad_face_features ? grad_face_features + (size_t)view_begin * num_faces * 3 * feat_dim : nullptr;
  // row-walk kernel: fp32 or bf16 features, D <= 4, rows a multiple of 4 px, a workspace with the face records
  float* acc = nullptr;
  int* job_ctr = nullptr;
  if (run_raster && feat_dim <= kRowWalkMaxD && (width % kRwSlab) == 0 && NF > 0) {
    const WorkspaceLayout L = workspace_layout({batch, NF, height, width, 0, false}, workspace, workspace_bytes_);
    if (L.fits) {
      acc = (float*)((char*)workspace + L.origin + L.face_records.at);
      job_ctr = (int*)((char*)workspace + L.origin + L.job_ctr(NFv, feat_dim).at);
    }
  }
  if (!(flags & DIBR_B200_ACCUMULATE) && !acc) {
    e = cudaMemsetAsync(g_xy_v, 0, (size_t)NFv * 6 * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
  }
  if (grad_face_features && feat_dim > 0 && (grad_features || !(flags & DIBR_B200_ACCUMULATE)) && !acc) {
    e = cudaMemsetAsync(g_ff_v, 0, (size_t)NFv * 3 * feat_dim * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
  }
  if (NF == 0) return 0;
  if (run_raster) {
    RasterBwdArgs a;
    const size_t px0 = (size_t)view_begin * height * width;
    a.B = nv; a.H = height; a.W = width; a.F = num_faces; a.D = feat_dim;
    a.ntx = (width + kTile - 1) / kTile; a.nty = (height + kTile - 1) / kTile;
    a.grad_feat = static_cast<const char*>(grad_features) + px0 * feat_dim * fsz;
    a.idx = face_idx + px0; a.w = output_weights ? output_weights + px0 * 3 : nullptr;
    a.xy = face_vertices_image + (size_t)view_begin * num_faces * 6;
    a.feat = static_cast<const char*>(face_features) + (size_t)view_begin * num_faces * 3 * feat_dim * fsz;
    a.grid = make_grid(multiplier, width, height); a.rc = make_raster_const(eps); a.multiplier = multiplier;
    a.grad_xy = g_xy_v;
    a.grad_feat_out = g_ff_v;
    if (acc) rc = bf16 ? launch_raster_bwd_rows<__nv_bfloat16>(a, acc, job_ctr, (flags & DIBR_B200_ACCUMULATE) ? 1 : 0, st)
                       : launch_raster_bwd_rows<float>(a, acc, job_ctr, (flags & DIBR_B200_ACCUMULATE) ? 1 : 0, st);
    else rc = bf16 ? launch_raster_bwd<__nv_bfloat16>(a, st) : launch_raster_bwd<float>(a, st);
    if (rc) return rc;
  }
  if (grad_soft_mask) {
    Scene& s = sa.s;
    s.xy = face_vertices_image;
    sa.sigmainv = sigmainv; sa.K = knum; sa.grad_soft = grad_soft_mask; sa.soft = soft_mask;
    sa.idx = face_idx; sa.grad_xy = grad_face_vertices_image;
    sa.view_begin = view_begin; sa.view_end = view_end;
    const unsigned persistent = persistent_grid(s, dibr_tile_soft_bwd_kernel);
    if (!bins_valid) {
      // no forward state: rebuild the large bins and recompute every tile
      rc = build_bins(s, 2, st);
      if (rc) return rc;
      sa.from_list = 0;
      Span sp("dibr_tile_soft_bwd_kernel<all tiles>", st);
      dibr_tile_soft_bwd_kernel<<<persistent, kThreads, 0, st>>>(sa);
    } else {
      // forward left the bins, the hit cache and the list of tiles it could not cache
      sa.from_list = 1;
      if (s.pool_tiles > 0) {
        Span sp("soft_bwd_runs_kernel", st);
        soft_bwd_runs_kernel<<<(unsigned)s.pool_tiles, kThreads, 0, st>>>(sa);
      }
      Span sp("dibr_tile_soft_bwd_kernel<leftovers>", st);
      dibr_tile_soft_bwd_kernel<<<persistent, kThreads, 0, st>>>(sa);
    }
    return (int)cudaGetLastError();
  }
  return 0;
}

int dibr_b200_backward(int batch, int num_faces, int height, int width, int feat_dim,
                       const float* grad_features, const float* grad_soft_mask,
                       const int64_t* face_idx, const float* output_weights, const float* soft_mask,
                       const float* face_vertices_image, const float* face_features,
                       float multiplier, float eps, float sigmainv, float boxlen_m, int knum,
                       float* grad_face_vertices_image, float* grad_face_features, void* workspace,
                       size_t workspace_bytes_, int flags, dibr_b200_stream_t stream) {
  return backward_impl(batch, num_faces, height, width, feat_dim, grad_features, grad_soft_mask, face_idx,
                       output_weights, soft_mask, face_vertices_image, face_features, multiplier, eps,
                       sigmainv, boxlen_m, knum, grad_face_vertices_image, grad_face_features, workspace,
                       workspace_bytes_, flags, stream, false, 0, batch);
}

int dibr_b200_backward_views(int batch, int num_faces, int height, int width, int feat_dim,
                             const void* grad_features, const float* grad_soft_mask,
                             const int64_t* face_idx, const float* output_weights, const float* soft_mask,
                             const float* face_vertices_image, const void* face_features, int features_bf16,
                             float multiplier, float eps, float sigmainv, float boxlen_m, int knum,
                             float* grad_face_vertices_image, float* grad_face_features, void* workspace,
                             size_t workspace_bytes_, int flags, int view_begin, int view_end,
                             dibr_b200_stream_t stream) {
  return backward_impl(batch, num_faces, height, width, feat_dim, grad_features, grad_soft_mask, face_idx,
                       output_weights, soft_mask, face_vertices_image, face_features, multiplier, eps,
                       sigmainv, boxlen_m, knum, grad_face_vertices_image, grad_face_features, workspace,
                       workspace_bytes_, flags, stream, features_bf16 != 0, view_begin, view_end);
}

int dibr_b200_backward_bf16(int batch, int num_faces, int height, int width, int feat_dim,
                            const uint16_t* grad_features, const float* grad_soft_mask,
                            const int64_t* face_idx, const float* output_weights, const float* soft_mask,
                            const float* face_vertices_image, const uint16_t* face_features,
                            float multiplier, float eps, float sigmainv, float boxlen_m, int knum,
                            float* grad_face_vertices_image, float* grad_face_features, void* workspace,
                            size_t workspace_bytes_, int flags, dibr_b200_stream_t stream) {
  return backward_impl(batch, num_faces, height, width, feat_dim, grad_features, grad_soft_mask, face_idx,
                       output_weights, soft_mask, face_vertices_image, face_features, multiplier, eps,
                       sigmainv, boxlen_m, knum, grad_face_vertices_image, grad_face_features, workspace,
                       workspace_bytes_, flags, stream, true, 0, batch);
}

int dibr_b200_packed_rasterize_forward(int batch, int64_t total_faces, int height, int width,
                                       int feat_dim, const float* face_vertices_z,
                                       const float* face_vertices_image, const float* face_bboxes,
                                       const float* face_features,
                                       const int64_t* first_idx_face_per_mesh, float multiplier,
                                       float eps, float* interpolated_features,
                                       int64_t* selected_face_idx, float* output_weights,
                                       void* workspace, size_t workspace_bytes_,
                                       dibr_b200_stream_t stream) {
  int rc = check_dims(batch, total_faces, height, width);
  if (rc) return rc;
  if (!selected_face_idx || !output_weights || !first_idx_face_per_mesh || feat_dim < 0) return DIBR_B200_EINVAL;
  if (feat_dim > 0 && (!interpolated_features || (total_faces > 0 && !face_features))) return DIBR_B200_EINVAL;
  if (total_faces > 0 && (!face_vertices_z || !face_vertices_image || !face_bboxes)) return DIBR_B200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  FwdArgs a;
  Scene& s = a.s;
  rc = setup_scene(s, batch, total_faces, 0, height, width, multiplier, 0.f, 0, false, workspace, workspace_bytes_);
  if (rc) return rc;
  s.first = first_idx_face_per_mesh; s.xy = face_vertices_image; s.z = face_vertices_z;
  s.premultiplied = 1; s.bbox_tight = face_bboxes;
  rc = build_bins(s, 1, st);
  if (rc) return rc;
  a.rc = make_raster_const(eps);
  a.D = feat_dim; a.feat = face_features; a.sigmainv = 0.f; a.K = 0;
  a.out_feat = interpolated_features; a.idx = selected_face_idx; a.out_w = output_weights; a.out_soft = nullptr;
  a.cache = 0;
  a.kl = SoftFwdOut{nullptr, nullptr, nullptr};
  launch_fwd<true, false, false>(a, st);
  return (int)cudaGetLastError();
}

int dibr_b200_rasterize_backward(int batch, int num_faces, int height, int width, int feat_dim,
                                 const float* grad_interpolated_features,
                                 const int64_t* selected_face_idx, const float* output_weights,
                                 const float* face_vertices_image, const float* face_features,
                                 float eps, float* grad_face_vertices_image,
                                 float* grad_face_features, dibr_b200_stream_t stream) {
  if (!grad_interpolated_features && feat_dim > 0) return DIBR_B200_EINVAL;
  // the packed forward's xy is premultiplied, so its weights cannot be recomputed here
  if (!output_weights && feat_dim > 0) return DIBR_B200_EINVAL;
  // workspace is not needed for the rasterize branch
  return dibr_b200_backward(batch, num_faces, height, width, feat_dim, grad_interpolated_features,
                            nullptr, selected_face_idx, output_weights, nullptr, face_vertices_image,
                            face_features, 1.f, eps, 0.f, 0.f, 0, grad_face_vertices_image,
                            grad_face_features, nullptr, 0, 0, stream);
}

int dibr_b200_soft_mask_forward(int batch, int num_faces, int height, int width, int knum,
                                const float* face_vertices_image, const float* face_large_bboxes,
                                const int64_t* selected_face_idx, float sigmainv, float multiplier,
                                float* soft_mask, float* close_face_prob, int64_t* close_face_idx,
                                uint8_t* close_face_dist_type, void* workspace,
                                size_t workspace_bytes_, dibr_b200_stream_t stream) {
  const int64_t NF = (int64_t)batch * num_faces;
  int rc = check_dims(batch, NF, height, width);
  if (rc) return rc;
  if (!selected_face_idx || !soft_mask || knum <= 0 || num_faces < 0) return DIBR_B200_EINVAL;
  if (num_faces > 0 && (!face_vertices_image || !face_large_bboxes)) return DIBR_B200_EINVAL;
  const bool lists = close_face_prob || close_face_idx || close_face_dist_type;
  if (lists && !(close_face_prob && close_face_idx && close_face_dist_type)) return DIBR_B200_EINVAL;
  if (lists && (int64_t)batch * height * width * knum < 0) return DIBR_B200_ESIZE;
  cudaStream_t st = (cudaStream_t)stream;
  FwdArgs a;
  Scene& s = a.s;
  rc = setup_scene(s, batch, NF, num_faces, height, width, multiplier, 0.f, 0, false, workspace, workspace_bytes_);
  if (rc) return rc;
  s.xy = face_vertices_image; s.premultiplied = 1; s.bbox_large = face_large_bboxes;
  rc = build_bins(s, 2, st);
  if (rc) return rc;
  a.rc = make_raster_const(0.f);
  a.D = 0; a.feat = nullptr; a.sigmainv = sigmainv; a.K = knum;
  a.out_feat = nullptr; a.idx = const_cast<int64_t*>(selected_face_idx); a.out_w = nullptr; a.out_soft = soft_mask;
  a.cache = 0;
  a.kl = SoftFwdOut{close_face_prob, close_face_idx, close_face_dist_type};
  if (lists) launch_fwd<false, true, true>(a, st);
  else launch_fwd<false, true, false>(a, st);
  return (int)cudaGetLastError();
}

int dibr_b200_soft_mask_backward(int batch, int num_faces, int height, int width, int knum,
                                 const float* grad_soft_mask, const float* soft_mask,
                                 const int64_t* selected_face_idx, const float* close_face_prob,
                                 const int64_t* close_face_idx, const uint8_t* close_face_dist_type,
                                 const float* face_vertices_image, float sigmainv, float multiplier,
                                 float* grad_face_vertices_image, dibr_b200_stream_t stream) {
  const int64_t NF = (int64_t)batch * num_faces;
  int rc = check_dims(batch, NF, height, width);
  if (rc) return rc;
  if (!grad_soft_mask || !soft_mask || !selected_face_idx || !close_face_prob || !close_face_idx ||
      !close_face_dist_type || !grad_face_vertices_image || knum <= 0 || !(multiplier > 0.f))
    return DIBR_B200_EINVAL;
  if (num_faces > 0 && !face_vertices_image) return DIBR_B200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(grad_face_vertices_image, 0, (size_t)NF * 6 * sizeof(float), st);
  if (e != cudaSuccess) return (int)e;
  if (NF == 0) return 0;
  SoftBwdListArgs a;
  a.B = batch; a.H = height; a.W = width; a.F = num_faces; a.K = knum;
  a.grid = make_grid(multiplier, width, height);
  a.sigmainv = sigmainv; a.multiplier = multiplier;
  a.grad_soft = grad_soft_mask; a.soft = soft_mask; a.idx = selected_face_idx;
  a.prob = close_face_prob; a.cidx = close_face_idx; a.ctype = close_face_dist_type;
  a.xy = face_vertices_image; a.grad_xy = grad_face_vertices_image;
  const int64_t P = (int64_t)batch * height * width;
  Span sp("soft_bwd_lists_kernel", st);
  soft_bwd_lists_kernel<<<(unsigned)((P + 255) / 256), 256, 0, st>>>(a);
  return (int)cudaGetLastError();
}

}  // extern "C"
