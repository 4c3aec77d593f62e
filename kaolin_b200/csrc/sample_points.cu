// sample_points.cu — H100 implementation of Kaolin's surface sampling and face areas
// (kaolin.ops.mesh.face_areas, packed_face_areas, sample_points, packed_sample_points;
// kaolin/ops/mesh/trianglemesh.py:30-311), behind the C ABI of include/dibr_b200.h.
//
// Views are ranges of one face array: view b owns the faces g in [face_off[b], face_off[b + 1]), reads
// face row g - b * fstride and vertex b * vstride + index.  Dense input (B, V, 3) with shared faces
// (F, 3) is fstride = F, vstride = V; packed input with merged faces is fstride = vstride = 0.
//
//   forward   sp_areas_kernel       one thread per face: the area with the reference's rounding (or the
//                                   given area), checked: an index outside [0, V) or an area that is
//                                   negative, NaN or infinite marks the view invalid;
//             sp_scan_tiles_kernel  per tile of kCdfTile faces, a segmented inclusive float64 scan (a view
//             sp_scan_carry_kernel  starts a segment), in place; one CTA scans the tile sums into carries;
//             sp_scan_apply_kernel  the carries are added, the coarse table (the CDF at every tile's last
//                                   face) written and a view whose total is not in (0, inf) marked.  Every
//                                   sum has a fixed order: the CDF does not depend on the run;
//             sp_sample_kernel      one thread per sample: Philox4x32-10, the face choice by a two-level
//                                   search (the view's coarse table in shared memory, then one CDF tile),
//                                   the gather and the interpolation.
//   backward  the samples grouped by face (count -> exclusive scan -> atomic-cursor fill -> row sort,
//             row_sort.cuh), then sp_face_grad_kernel sums each face's w_k * g in ascending sample order
//             (the Philox uniforms are recomputed, not stored) into the face_features gradient and the
//             per-corner vertex gradients, and sp_gather_kernel adds every vertex's corners over the
//             corner CSR of the mesh topology (csrc/mesh_topology.cu).  No float atomics.
//
// The random stream (DESIGN.md, f15): key (k0, k1) = the two halves of a 64-bit device word; sample n
// of view b uses the Philox4x32-10 blocks of counter (n, 0, b, j).  float32: block 0 gives r from words
// 0 and 1, u from word 2 and v from word 3; float64: block 0 gives r and u, block 1 gives v.  r is
// always ((w_a << 21) | (w_b >> 11)) * 2^-53; float32 u, v are (w >> 8) * 2^-24, float64 u, v take the
// 53-bit form.  The face is the smallest f with c_f > t, t = r * c_last; if rounding makes t reach
// c_last, the first f with c_f = c_last.  A zero-area face is never chosen.
//
// Rounding is the reference's, every operation rounded on its own (nvcc would contract to FMA):
//   area   x = v0 - v1, y = v1 - v2; sqrt((a + b) + c) * 0.5 with a = (x2*y3 - x3*y2)^2 and cyclic
//   point  u = sqrt(u_raw), w0 = 1 - u, w1 = u * (1 - v), w2 = u * v; p = (w0*v0 + w1*v1) + w2*v2
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>

#include "../../include/dibr_b200.h"
#include "op_layouts.h"
#include "row_sort.cuh"
#include "scan.cuh"

// launch tracing (dibr_b200_trace_begin / _end), kept in dibr_b200.cu
namespace dibr_b200_detail {
bool span_open(const char* name, cudaStream_t st);
void span_close(cudaStream_t st);
}  // namespace dibr_b200_detail

namespace {

struct Span {
  cudaStream_t st;
  bool on;
  Span(const char* name, cudaStream_t st_) : st(st_), on(dibr_b200_detail::span_open(name, st_)) {}
  ~Span() { if (on) dibr_b200_detail::span_close(st); }
};

using dibr_b200_detail::exclusive_scan;
using dibr_layout::carve;
using dibr_layout::kCdfTile;
using dibr_layout::piece;

constexpr int kThreads = 256;
constexpr int kScanItems = kCdfTile / kThreads;          // faces per thread of sp_scan_tiles_kernel
constexpr int kCarryThreads = 1024;
constexpr int kSamplesPerThread = 4;
constexpr int kSamplesPerCta = kThreads * kSamplesPerThread;
constexpr int kCoarseSmem = 6144;                        // coarse entries staged in shared memory (48 KB)
constexpr int kFeatureChunk = 4;                         // feature channels summed per pass of a face's row
constexpr int kShortRow = 32;                            // rows of at most this many samples: one thread sorts
constexpr int kLongCtas = 132;
constexpr int kSortThreads = 1024;
static_assert(kCdfTile % kThreads == 0, "whole items per thread");

// Correctly rounded operations, never contracted.
template <typename T> struct Rn;
template <> struct Rn<float> {
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float div(float a, float b) { return __fdiv_rn(a, b); }
  static __device__ __forceinline__ float sqrt(float a) { return __fsqrt_rn(a); }
};
template <> struct Rn<double> {
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
  static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
  static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
  static __device__ __forceinline__ double div(double a, double b) { return __ddiv_rn(a, b); }
  static __device__ __forceinline__ double sqrt(double a) { return __dsqrt_rn(a); }
};

template <typename T> __device__ __forceinline__ T qnan() { return (T)__int_as_float(0x7fffffff); }

// The views of one call (see the top of the file).
struct Views {
  int B, V;              // V: the bound of a face index
  int64_t nf, fstride, vstride;
  const int64_t* face_off;   // [B + 1]
  const int64_t* faces;
};

// The view of face g: the largest b with face_off[b] <= g (empty views own no face).
__device__ __forceinline__ int view_of(const Views& m, int64_t g) {
  int lo = 0, hi = m.B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(m.face_off + mid) <= g) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// The three corners of face g of view b; false (nothing read) when an index is outside [0, V).
template <typename T>
__device__ __forceinline__ bool load_face(const Views& m, const T* __restrict__ vertices, int b, int64_t g, T v[3][3]) {
  const int64_t* row = m.faces + (g - b * m.fstride) * 3;
  int64_t idx[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    idx[k] = __ldg(row + k);
    if (idx[k] < 0 || idx[k] >= m.V) return false;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const T* p = vertices + (b * m.vstride + idx[k]) * 3;
    v[k][0] = __ldg(p); v[k][1] = __ldg(p + 1); v[k][2] = __ldg(p + 2);
  }
  return true;
}

// trianglemesh.py:30-40 with its rounding.
template <typename T>
__device__ __forceinline__ T face_area(const T v[3][3]) {
  using R = Rn<T>;
  T x[3], y[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) { x[c] = R::sub(v[0][c], v[1][c]); y[c] = R::sub(v[1][c], v[2][c]); }
  const T A = R::sub(R::mul(x[1], y[2]), R::mul(x[2], y[1]));
  const T B = R::sub(R::mul(x[2], y[0]), R::mul(x[0], y[2]));
  const T C = R::sub(R::mul(x[0], y[1]), R::mul(x[1], y[0]));
  return R::mul(R::sqrt(R::add(R::add(R::mul(A, A), R::mul(B, B)), R::mul(C, C))), T(0.5));
}

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 and the random stream.

struct U4 { uint32_t w[4]; };

__device__ __forceinline__ U4 philox(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * c0, hi0 = __umulhi(0xD2511F53u, c0);
    const uint32_t lo1 = 0xCD9E8D57u * c2, hi1 = __umulhi(0xCD9E8D57u, c2);
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return {{c0, c1, c2, c3}};
}

__device__ __forceinline__ double u53(uint32_t a, uint32_t b) {
  return (double)((((uint64_t)a) << 21) | (b >> 11)) * 0x1p-53;
}
__device__ __forceinline__ float u24(uint32_t w) { return (float)(w >> 8) * 0x1p-24f; }

template <typename T> struct Stream;
template <> struct Stream<float> {
  static __device__ __forceinline__ void draw(uint32_t n, uint32_t b, uint32_t k0, uint32_t k1, double& r, float& u,
                                              float& v) {
    const U4 w = philox(n, 0u, b, 0u, k0, k1);
    r = u53(w.w[0], w.w[1]); u = u24(w.w[2]); v = u24(w.w[3]);
  }
};
template <> struct Stream<double> {
  static __device__ __forceinline__ void draw(uint32_t n, uint32_t b, uint32_t k0, uint32_t k1, double& r, double& u,
                                              double& v) {
    const U4 w = philox(n, 0u, b, 0u, k0, k1), x = philox(n, 0u, b, 1u, k0, k1);
    r = u53(w.w[0], w.w[1]); u = u53(w.w[2], w.w[3]); v = u53(x.w[0], x.w[1]);
  }
};

// The barycentric weights of trianglemesh.py:76-85.
template <typename T>
__device__ __forceinline__ void weights(T u_raw, T v, T w[3]) {
  using R = Rn<T>;
  const T u = R::sqrt(u_raw);
  w[0] = R::sub(T(1), u);
  w[1] = R::mul(u, R::sub(T(1), v));
  w[2] = R::mul(u, v);
}

// (w0*a0 + w1*a1) + w2*a2
template <typename T>
__device__ __forceinline__ T interp(const T w[3], T a0, T a1, T a2) {
  using R = Rn<T>;
  return R::add(R::add(R::mul(w[0], a0), R::mul(w[1], a1)), R::mul(w[2], a2));
}

// ---------------------------------------------------------------------------------------------
// Forward.

// areas_out (optional) gets the computed area; cdf (optional) the float64 area to scan; with
// view_flag, a bad index or an area outside [0, inf) marks the view.
template <typename T>
__global__ void __launch_bounds__(kThreads) sp_areas_kernel(Views m, const T* __restrict__ vertices,
                                                            const double* __restrict__ given, T* __restrict__ areas_out,
                                                            double* __restrict__ cdf, int* __restrict__ view_flag,
                                                            int* __restrict__ status) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= m.nf) return;
  const int b = view_of(m, g);
  T v[3][3];
  const bool ok = load_face(m, vertices, b, g, v);
  if (!ok) atomicOr(status, DIBR_B200_SAMPLE_BAD_INDEX);
  double a;
  if (given) {
    a = given[g];
  } else {
    const T ar = ok ? face_area(v) : qnan<T>();
    if (areas_out) areas_out[g] = ar;
    a = (double)ar;
  }
  if (cdf) cdf[g] = a;
  if (view_flag && (!ok || !(a >= 0.0 && a <= DBL_MAX))) {
    atomicOr(view_flag + b, 1);
    atomicOr(status, DIBR_B200_SAMPLE_BAD_DISTRIBUTION);
  }
}

// (starts a view, sum) pairs under the segmented-scan operator: l then r.
struct Seg { int f; double s; };
__device__ __forceinline__ Seg combine(Seg l, Seg r) { return {l.f | r.f, r.f ? r.s : __dadd_rn(l.s, r.s)}; }
__device__ __forceinline__ Seg shfl_up(Seg x, int d) {
  return {__shfl_up_sync(0xffffffffu, x.f, d), __shfl_up_sync(0xffffffffu, x.s, d)};
}

// Inclusive segmented scan of one pair per thread across the CTA (blockDim.x a multiple of 32, at
// most 1024); *excl gets the thread's exclusive prefix ({0, 0} for thread 0), *total the CTA's.
__device__ Seg block_seg_scan(Seg x, Seg* excl, Seg* total) {
  __shared__ int sf[32];
  __shared__ double ss[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const Seg y = shfl_up(x, d);
    if (lane >= d) x = combine(y, x);
  }
  if (lane == 31) { sf[warp] = x.f; ss[warp] = x.s; }
  __syncthreads();
  if (warp == 0) {
    Seg w = lane < nwarps ? Seg{sf[lane], ss[lane]} : Seg{0, 0.0};
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const Seg y = shfl_up(w, d);
      if (lane >= d) w = combine(y, w);
    }
    if (lane < nwarps) { sf[lane] = w.f; ss[lane] = w.s; }
  }
  __syncthreads();
  const Seg before = warp ? Seg{sf[warp - 1], ss[warp - 1]} : Seg{0, 0.0};
  const Seg inc = warp ? combine(before, x) : x;
  Seg ex = shfl_up(inc, 1);
  if (lane == 0) ex = before;
  *excl = ex;
  *total = {sf[nwarps - 1], ss[nwarps - 1]};
  __syncthreads();   // sf, ss are reused by the next call
  return inc;
}

// Tile blockIdx.x: each thread scans kScanItems consecutive faces, then the CTA adds the prefix of the
// threads before to the faces ahead of each thread's first view start.
__global__ void __launch_bounds__(kThreads) sp_scan_tiles_kernel(Views m, double* __restrict__ cdf,
                                                                 double* __restrict__ tile_sum, int* __restrict__ tile_flag) {
  const int64_t base = (int64_t)blockIdx.x * kCdfTile + (int64_t)threadIdx.x * kScanItems;
  double val[kScanItems];
  int first = kScanItems;   // the thread's first item that starts a view
  Seg own = {0, 0.0};
  if (base < m.nf) {
    int b = view_of(m, base);
    int64_t next = __ldg(m.face_off + b + 1);
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) {
      const int64_t g = base + i;
      if (g >= m.nf) { val[i] = 0.0; continue; }
      while (next <= g) { ++b; next = __ldg(m.face_off + b + 1); }
      const bool start = g == __ldg(m.face_off + b);
      const double a = cdf[g];
      own.s = start ? a : __dadd_rn(own.s, a);
      if (start && first == kScanItems) first = i;
      own.f |= start;
      val[i] = own.s;
    }
  }
  Seg excl, total;
  block_seg_scan(own, &excl, &total);
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    const int64_t g = base + i;
    if (g < m.nf) cdf[g] = i < first ? __dadd_rn(excl.s, val[i]) : val[i];
  }
  if (threadIdx.x == 0) { tile_sum[blockIdx.x] = total.s; tile_flag[blockIdx.x] = total.f; }
}

// One CTA: carry[k] = the segmented sum of the tiles before k, in tile order; an empty view is invalid.
__global__ void __launch_bounds__(kCarryThreads) sp_scan_carry_kernel(Views m, int64_t tiles,
                                                                      const double* __restrict__ tile_sum,
                                                                      const int* __restrict__ tile_flag,
                                                                      double* __restrict__ carry, int* __restrict__ view_flag,
                                                                      int* __restrict__ status) {
  for (int b = threadIdx.x; b < m.B; b += blockDim.x)
    if (m.face_off[b + 1] == m.face_off[b]) {
      atomicOr(view_flag + b, 1);
      atomicOr(status, DIBR_B200_SAMPLE_BAD_DISTRIBUTION);
    }
  Seg run = {0, 0.0};
  for (int64_t k0 = 0; k0 < tiles; k0 += blockDim.x) {
    const int64_t k = k0 + threadIdx.x;
    const Seg x = k < tiles ? Seg{tile_flag[k], tile_sum[k]} : Seg{0, 0.0};
    Seg excl, total;
    block_seg_scan(x, &excl, &total);
    if (k < tiles) carry[k] = (threadIdx.x ? combine(run, excl) : run).s;
    run = combine(run, total);
  }
}

// The carries, the coarse table and the check of each view's total.
__global__ void __launch_bounds__(kThreads) sp_scan_apply_kernel(Views m, const double* __restrict__ carry,
                                                                 double* __restrict__ cdf, double* __restrict__ coarse,
                                                                 int* __restrict__ view_flag, int* __restrict__ status) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= m.nf) return;
  const int64_t k = g / kCdfTile;
  const int b = view_of(m, g);
  double c = cdf[g];
  if (__ldg(m.face_off + b) < k * kCdfTile) {
    c = __dadd_rn(carry[k], c);
    cdf[g] = c;
  }
  if (g == (k + 1) * kCdfTile - 1) coarse[k] = c;
  if (g == __ldg(m.face_off + b + 1) - 1 && !(c > 0.0 && c <= DBL_MAX)) {
    atomicOr(view_flag + b, 1);
    atomicOr(status, DIBR_B200_SAMPLE_BAD_DISTRIBUTION);
  }
}

// The smallest i in [lo, hi) with a[i] > t (strict) or a[i] >= t; hi if none.
__device__ __forceinline__ int64_t lower(const double* a, int64_t lo, int64_t hi, double t, bool strict) {
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    const double x = a[mid];
    if (strict ? x > t : x >= t) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// CTA blockIdx.x: view blockIdx.x / nblk, samples (blockIdx.x % nblk) * kSamplesPerCta + j * kThreads +
// threadIdx.x.  The coarse table of the view's tiles but the last is staged in shared memory when it
// holds at most `smem_coarse` entries, else searched in place.
template <typename T>
__global__ void __launch_bounds__(kThreads) sp_sample_kernel(Views m, int N, int D, int nblk, int smem_coarse,
                                                             const T* __restrict__ vertices,
                                                             const T* __restrict__ face_features,
                                                             const int64_t* __restrict__ key,
                                                             const double* __restrict__ cdf,
                                                             const double* __restrict__ coarse,
                                                             const int* __restrict__ view_flag, T* __restrict__ points,
                                                             int64_t* __restrict__ choices, T* __restrict__ features) {
  extern __shared__ double s_coarse[];
  const int b = blockIdx.x / nblk;
  const int n0 = (blockIdx.x % nblk) * kSamplesPerCta;
  const int64_t s = __ldg(m.face_off + b), e = __ldg(m.face_off + b + 1);
  const bool bad = __ldg(view_flag + b) != 0;
  const int64_t ks = s / kCdfTile;
  const int64_t nc = bad ? 0 : (e - 1) / kCdfTile - ks;   // tiles of the view before its last
  const double* cs = coarse + ks;
  if (nc <= smem_coarse) {
    for (int64_t i = threadIdx.x; i < nc; i += kThreads) s_coarse[i] = cs[i];
    __syncthreads();
    cs = s_coarse;
  }
  const uint64_t k64 = (uint64_t)__ldg(key);
  const uint32_t k0 = (uint32_t)k64, k1 = (uint32_t)(k64 >> 32);
  const double last = bad ? 0.0 : cdf[e - 1];
#pragma unroll 1
  for (int j = 0; j < kSamplesPerThread; ++j) {
    const int n = n0 + j * kThreads + threadIdx.x;
    if (n >= N) break;
    const int64_t o = (int64_t)b * N + n;
    T v[3][3];
    T w[3];
    int64_t g = -1;
    bool ok = false;
    if (!bad) {
      double r;
      T u, vv;
      Stream<T>::draw((uint32_t)n, (uint32_t)b, k0, k1, r, u, vv);
      double t = __dmul_rn(r, last);
      const bool strict = t < last;
      if (!strict) t = last;
      const int64_t tile = ks + lower(cs, 0, nc, t, strict);
      const int64_t lo = tile * kCdfTile > s ? tile * kCdfTile : s;
      const int64_t hi = (tile + 1) * kCdfTile < e ? (tile + 1) * kCdfTile : e;
      g = lower(cdf, lo, hi, t, strict);
      if (g >= e) g = e - 1;
      weights(u, vv, w);
      ok = load_face(m, vertices, b, g, v);
    }
    choices[o] = g < 0 ? -1 : g - b * m.fstride;
#pragma unroll
    for (int c = 0; c < 3; ++c) points[o * 3 + c] = ok ? interp(w, v[0][c], v[1][c], v[2][c]) : qnan<T>();
    if (features) {
      const T* f = face_features + g * 3 * D;
      for (int d = 0; d < D; ++d)
        features[o * D + d] = ok ? interp(w, __ldg(f + d), __ldg(f + D + d), __ldg(f + 2 * D + d)) : qnan<T>();
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Backward.

__global__ void __launch_bounds__(kThreads) sp_count_kernel(int N, int64_t np, int64_t fstride,
                                                            const int64_t* __restrict__ choices, int* __restrict__ count) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= np) return;
  const int64_t f = choices[i];
  if (f >= 0) atomicAdd(count + f + (i / N) * fstride, 1);
}

// Each sample takes a slot of its face's row in whatever order the atomics give; the row sort puts the
// sample ids in ascending order.
__global__ void __launch_bounds__(kThreads) sp_fill_kernel(int N, int64_t np, int64_t fstride,
                                                           const int64_t* __restrict__ choices, const int* __restrict__ off,
                                                           int* __restrict__ count, int* __restrict__ ids) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= np) return;
  const int64_t f = choices[i];
  if (f < 0) return;
  const int64_t b = i / N, row = f + b * fstride;
  ids[off[row] + atomicSub(count + row, 1) - 1] = (int)(i - b * N);
}

__global__ void __launch_bounds__(kThreads) sp_sort_rows_kernel(int64_t rows, const int* __restrict__ off,
                                                                int* __restrict__ ids, int* __restrict__ long_rows,
                                                                int* __restrict__ long_count) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int b = off[r], n = off[r + 1] - b;
  if (n > kShortRow) {
    long_rows[atomicAdd(long_count, 1)] = (int)r;
    return;
  }
  insertion_sort(ids + b, n);
}

__global__ void __launch_bounds__(kSortThreads) sp_sort_long_kernel(const int* __restrict__ off, int* __restrict__ ids,
                                                                    const int* __restrict__ long_rows,
                                                                    const int* __restrict__ long_count) {
  const int rows = *long_count;
  for (int k = blockIdx.x; k < rows; k += gridDim.x) {
    const int r = long_rows[k];
    block_bitonic_sort(ids + off[r], off[r + 1] - off[r]);
  }
}

// One thread per face g: over its samples in ascending order, corner k's gradients are
// sum(w_k * grad_points) (corner_grad [nf][3][3], when given) and sum(w_k * grad_features)
// (grad_ff [nf][3][D], when given), each product rounded and added from 0 as the reference's
// scatter_add does.  A face no sample chose gets zeros.
template <typename T>
__global__ void __launch_bounds__(kThreads) sp_face_grad_kernel(Views m, int N, int D, const int64_t* __restrict__ key,
                                                                const int* __restrict__ off, const int* __restrict__ ids,
                                                                const T* __restrict__ grad_points,
                                                                const T* __restrict__ grad_features,
                                                                T* __restrict__ corner_grad, T* __restrict__ grad_ff) {
  using R = Rn<T>;
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= m.nf) return;
  const int b = view_of(m, g);
  const int r0 = off[g], r1 = off[g + 1];
  const uint64_t k64 = (uint64_t)__ldg(key);
  const uint32_t k0 = (uint32_t)k64, k1 = (uint32_t)(k64 >> 32);
  const int chunks = grad_ff ? (D + kFeatureChunk - 1) / kFeatureChunk : 0;
  const int passes = corner_grad && chunks == 0 ? 1 : chunks;
  for (int p = 0; p < passes; ++p) {
    const bool verts = corner_grad && p == 0;
    const int d0 = p * kFeatureChunk;
    T av[3][3] = {}, af[3][kFeatureChunk] = {};
    for (int q = r0; q < r1; ++q) {
      const int n = ids[q];
      double r;
      T u, v, w[3];
      Stream<T>::draw((uint32_t)n, (uint32_t)b, k0, k1, r, u, v);
      weights(u, v, w);
      const int64_t o = (int64_t)b * N + n;
      if (verts) {
        T gp[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) gp[c] = grad_points[o * 3 + c];
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
          for (int c = 0; c < 3; ++c) av[k][c] = R::add(av[k][c], R::mul(w[k], gp[c]));
      }
      if (grad_ff) {
#pragma unroll
        for (int dd = 0; dd < kFeatureChunk; ++dd) {
          if (d0 + dd >= D) break;
          const T gf = grad_features[o * D + d0 + dd];
#pragma unroll
          for (int k = 0; k < 3; ++k) af[k][dd] = R::add(af[k][dd], R::mul(w[k], gf));
        }
      }
    }
    if (verts)
#pragma unroll
      for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int c = 0; c < 3; ++c) corner_grad[g * 9 + k * 3 + c] = av[k][c];
    if (grad_ff)
#pragma unroll
      for (int dd = 0; dd < kFeatureChunk; ++dd) {
        if (d0 + dd >= D) break;
#pragma unroll
        for (int k = 0; k < 3; ++k) grad_ff[(g * 3 + k) * D + d0 + dd] = af[k][dd];
      }
  }
}

// The reference's autograd of face_area (sqrt, pow 2, products), per corner, into corner_grad [nf][3][3].
// A zero-area face gives NaN, as the reference's does.
template <typename T>
__global__ void __launch_bounds__(kThreads) sp_area_grad_kernel(Views m, const T* __restrict__ vertices,
                                                                const T* __restrict__ grad_areas, T* __restrict__ corner_grad) {
  using R = Rn<T>;
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= m.nf) return;
  const int b = view_of(m, g);
  T v[3][3];
  T* o = corner_grad + g * 9;
  if (!load_face(m, vertices, b, g, v)) {
    for (int k = 0; k < 9; ++k) o[k] = T(0);
    return;
  }
  T x[3], y[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) { x[c] = R::sub(v[0][c], v[1][c]); y[c] = R::sub(v[1][c], v[2][c]); }
  const T A = R::sub(R::mul(x[1], y[2]), R::mul(x[2], y[1]));
  const T B = R::sub(R::mul(x[2], y[0]), R::mul(x[0], y[2]));
  const T C = R::sub(R::mul(x[0], y[1]), R::mul(x[1], y[0]));
  const T root = R::sqrt(R::add(R::add(R::mul(A, A), R::mul(B, B)), R::mul(C, C)));
  const T gsum = R::div(R::mul(grad_areas[g], T(0.5)), R::mul(T(2), root));
  const T gA = R::mul(gsum, R::mul(T(2), A)), gB = R::mul(gsum, R::mul(T(2), B)), gC = R::mul(gsum, R::mul(T(2), C));
  T gx[3], gy[3];
  gx[0] = R::sub(R::mul(gC, y[1]), R::mul(gB, y[2]));
  gx[1] = R::sub(R::mul(gA, y[2]), R::mul(gC, y[0]));
  gx[2] = R::sub(R::mul(gB, y[0]), R::mul(gA, y[1]));
  gy[0] = R::sub(R::mul(gB, x[2]), R::mul(gC, x[1]));
  gy[1] = R::sub(R::mul(gC, x[0]), R::mul(gA, x[2]));
  gy[2] = R::sub(R::mul(gA, x[1]), R::mul(gB, x[0]));
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    o[c] = gx[c];
    o[3 + c] = R::sub(gy[c], gx[c]);
    o[6 + c] = -gy[c];
  }
}

// grad_vertices[b, v, c] = the sum over v's corners (corner CSR order) of corner_grad[b * cstride + corner][c],
// for `views` views of V vertices; every element is written.
template <typename T>
__global__ void __launch_bounds__(kThreads) sp_gather_kernel(int64_t total, int V, int64_t cstride,
                                                             const int* __restrict__ corner_ptr,
                                                             const int* __restrict__ corners,
                                                             const T* __restrict__ corner_grad, T* __restrict__ out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int64_t r = t / 3;
  const int c = (int)(t - r * 3);
  const int64_t b = r / V;
  const int v = (int)(r - b * V);
  const T* src = corner_grad + b * cstride * 3 + c;
  T s = T(0);
  for (int p = __ldg(corner_ptr + v); p < __ldg(corner_ptr + v + 1); ++p)
    s = Rn<T>::add(s, __ldg(src + (int64_t)__ldg(corners + p) * 3));
  out[t] = s;
}

// ---------------------------------------------------------------------------------------------
// Host.

unsigned blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

size_t tsize_of(int dtype) {
  return dtype == DIBR_B200_DTYPE_F32 ? sizeof(float) : dtype == DIBR_B200_DTYPE_F64 ? sizeof(double) : 0;
}

// 0 or the error: every corner (3 * nf) and every (view, sample) index fits an int.
int check_dims(int B, int64_t nf, int N, int dtype) {
  if (B < 0 || nf < 0 || N < 0 || tsize_of(dtype) == 0) return DIBR_B200_EINVAL;
  if (3 * nf >= 0x7fffffffLL || (int64_t)B * N >= 0x7fffffffLL) return DIBR_B200_ESIZE;
  return 0;
}

Views views(int B, int64_t nf, int V, int64_t fstride, int64_t vstride, const int64_t* face_off, const int64_t* faces) {
  return Views{B, V, nf, fstride, vstride, face_off, faces};
}

template <typename T>
int sample_forward(const Views& m, int N, int D, const T* vertices, const double* given, const T* ff, const int64_t* key,
                   T* points, int64_t* choices, T* features, int* status, char* o,
                   const dibr_layout::SamplePointsForwardLayout& L, cudaStream_t st) {
  double* cdf = piece<double>(o, L.cdf);
  double* coarse = piece<double>(o, L.coarse);
  double* carry = piece<double>(o, L.carry);
  int* view_flag = piece<int>(o, L.view_flag);
  const int64_t tiles = dibr_layout::cdf_tiles(m.nf);
  cudaError_t e = cudaMemsetAsync(view_flag, 0, sizeof(int) * (size_t)m.B, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(status, 0, sizeof(int), st);
  if (e != cudaSuccess) return (int)e;
  {
    Span sp("sp_areas_kernel", st);
    sp_areas_kernel<T><<<blocks(m.nf, kThreads), kThreads, 0, st>>>(m, vertices, given, nullptr, cdf, view_flag, status);
  }
  {
    Span sp("sp_scan_kernels", st);
    sp_scan_tiles_kernel<<<(unsigned)tiles, kThreads, 0, st>>>(m, cdf, piece<double>(o, L.tile_sum),
                                                               piece<int>(o, L.tile_flag));
    sp_scan_carry_kernel<<<1, kCarryThreads, 0, st>>>(m, tiles, piece<double>(o, L.tile_sum), piece<int>(o, L.tile_flag),
                                                      carry, view_flag, status);
    sp_scan_apply_kernel<<<blocks(m.nf, kThreads), kThreads, 0, st>>>(m, carry, cdf, coarse, view_flag, status);
  }
  if (N > 0) {
    Span sp("sp_sample_kernel", st);
    const int nblk = (N + kSamplesPerCta - 1) / kSamplesPerCta;
    const int smem_coarse = (int)(tiles < kCoarseSmem ? tiles : kCoarseSmem);
    sp_sample_kernel<T><<<(unsigned)((int64_t)m.B * nblk), kThreads, sizeof(double) * (size_t)smem_coarse, st>>>(
        m, N, D, nblk, smem_coarse, vertices, ff, key, cdf, coarse, view_flag, points, choices, features);
  }
  return (int)cudaGetLastError();
}

template <typename T>
int gather(int views_n, int V, int64_t cstride, const int* corner_ptr, const int* corners, const T* corner_grad,
           T* grad_vertices, cudaStream_t st) {
  const int64_t total = (int64_t)views_n * V * 3;
  Span sp("sp_gather_kernel", st);
  if (total > 0)
    sp_gather_kernel<T><<<blocks(total, kThreads), kThreads, 0, st>>>(total, V, cstride, corner_ptr, corners, corner_grad,
                                                                      grad_vertices);
  return (int)cudaGetLastError();
}

template <typename T>
int sample_backward(const Views& m, int N, int D, const int64_t* key, const int64_t* choices, const T* grad_points,
                    const T* grad_features, const int* corner_ptr, const int* corners, T* grad_vertices, T* grad_ff,
                    char* o, const dibr_layout::SamplePointsBackwardLayout& L, cudaStream_t st) {
  const int64_t np = (int64_t)m.B * N, rows = m.nf;
  int* count = piece<int>(o, L.count);
  int* off = piece<int>(o, L.off);
  int* ids = piece<int>(o, L.ids);
  int* long_rows = piece<int>(o, L.long_rows);
  int* long_count = piece<int>(o, L.long_count);
  T* corner_grad = grad_vertices ? piece<T>(o, L.corner_grad) : nullptr;
  cudaError_t e = cudaMemsetAsync(count, 0, sizeof(int) * (size_t)rows, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(long_count, 0, sizeof(int), st);
  if (e != cudaSuccess) return (int)e;
  {
    Span sp("sp_group_kernels", st);
    if (np > 0) sp_count_kernel<<<blocks(np, kThreads), kThreads, 0, st>>>(N, np, m.fstride, choices, count);
    if (int r = exclusive_scan(count, (int)rows, piece<int>(o, L.sums), off, st)) return r;
    if (np > 0) sp_fill_kernel<<<blocks(np, kThreads), kThreads, 0, st>>>(N, np, m.fstride, choices, off, count, ids);
    sp_sort_rows_kernel<<<blocks(rows, kThreads), kThreads, 0, st>>>(rows, off, ids, long_rows, long_count);
    sp_sort_long_kernel<<<kLongCtas, kSortThreads, 0, st>>>(off, ids, long_rows, long_count);
  }
  {
    Span sp("sp_face_grad_kernel", st);
    sp_face_grad_kernel<T><<<blocks(rows, kThreads), kThreads, 0, st>>>(m, N, D, key, off, ids, grad_points,
                                                                         grad_features, corner_grad, grad_ff);
  }
  if (!grad_vertices) return (int)cudaGetLastError();
  return gather<T>(m.vstride ? m.B : 1, m.V, m.fstride * 3, corner_ptr, corners, corner_grad, grad_vertices, st);
}

}  // namespace

extern "C" {

int dibr_b200_sample_points_workspace_bytes(int batch, int64_t total_faces, int num_samples, int dtype,
                                            size_t* forward_bytes, size_t* backward_bytes) {
  if (int r = check_dims(batch, total_faces, num_samples, dtype)) return r;
  if (forward_bytes) *forward_bytes = dibr_layout::sample_points_forward_layout(batch, total_faces).bytes;
  if (backward_bytes)
    *backward_bytes = dibr_layout::sample_points_backward_layout(batch, total_faces, num_samples, tsize_of(dtype)).bytes;
  return 0;
}

int dibr_b200_face_areas_forward(int batch, int64_t total_faces, int num_vertices, int64_t fstride, int64_t vstride,
                                 int dtype, const int64_t* face_off, const int64_t* faces, const void* vertices,
                                 void* areas, int32_t* status, dibr_b200_stream_t stream) {
  if (int r = check_dims(batch, total_faces, 0, dtype)) return r;
  if (num_vertices < 0 || !status || (total_faces > 0 && (batch < 1 || !face_off || !faces || !vertices || !areas)))
    return DIBR_B200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(status, 0, sizeof(int), st);
  if (e != cudaSuccess) return (int)e;
  if (total_faces == 0) return 0;
  const Views m = views(batch, total_faces, num_vertices, fstride, vstride, face_off, faces);
  Span sp("sp_areas_kernel", st);
  if (dtype == DIBR_B200_DTYPE_F32)
    sp_areas_kernel<float><<<blocks(total_faces, kThreads), kThreads, 0, st>>>(m, (const float*)vertices, nullptr,
                                                                                (float*)areas, nullptr, nullptr, status);
  else
    sp_areas_kernel<double><<<blocks(total_faces, kThreads), kThreads, 0, st>>>(m, (const double*)vertices, nullptr,
                                                                                 (double*)areas, nullptr, nullptr, status);
  return (int)cudaGetLastError();
}

int dibr_b200_face_areas_backward(int batch, int64_t total_faces, int num_vertices, int64_t fstride, int64_t vstride,
                                  int dtype, const int64_t* face_off, const int64_t* faces, const void* vertices,
                                  const void* grad_areas, const int32_t* corner_ptr, const int32_t* corners,
                                  void* grad_vertices, void* workspace, size_t workspace_bytes,
                                  dibr_b200_stream_t stream) {
  if (int r = check_dims(batch, total_faces, 0, dtype)) return r;
  if (num_vertices < 0 || !workspace || !grad_vertices || !corner_ptr ||
      (total_faces > 0 && (batch < 1 || !face_off || !faces || !vertices || !grad_areas || !corners)))
    return DIBR_B200_EINVAL;
  const dibr_layout::SamplePointsBackwardLayout L =
      dibr_layout::sample_points_backward_layout(batch, total_faces, 0, tsize_of(dtype));
  char* o = carve(workspace, workspace_bytes, L.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const Views m = views(batch, total_faces, num_vertices, fstride, vstride, face_off, faces);
  const int nviews = vstride ? batch : 1;
  if (dtype == DIBR_B200_DTYPE_F32) {
    float* cg = piece<float>(o, L.corner_grad);
    if (total_faces > 0)
      sp_area_grad_kernel<float><<<blocks(total_faces, kThreads), kThreads, 0, st>>>(m, (const float*)vertices,
                                                                                      (const float*)grad_areas, cg);
    return gather<float>(nviews, num_vertices, fstride * 3, corner_ptr, corners, cg, (float*)grad_vertices, st);
  }
  double* cg = piece<double>(o, L.corner_grad);
  if (total_faces > 0)
    sp_area_grad_kernel<double><<<blocks(total_faces, kThreads), kThreads, 0, st>>>(m, (const double*)vertices,
                                                                                     (const double*)grad_areas, cg);
  return gather<double>(nviews, num_vertices, fstride * 3, corner_ptr, corners, cg, (double*)grad_vertices, st);
}

int dibr_b200_sample_points_forward(int batch, int64_t total_faces, int num_vertices, int64_t fstride, int64_t vstride,
                                    int dtype, int num_samples, int feature_dim, const int64_t* face_off,
                                    const int64_t* faces, const void* vertices, const double* areas,
                                    const void* face_features, const int64_t* key, void* points,
                                    int64_t* face_choices, void* features, int32_t* status, void* workspace,
                                    size_t workspace_bytes, dibr_b200_stream_t stream) {
  if (int r = check_dims(batch, total_faces, num_samples, dtype)) return r;
  if (num_vertices < 0 || feature_dim < 0 || (face_features != nullptr) != (features != nullptr) ||
      (face_features && fstride == 0) || !status || !workspace || batch < 1 || total_faces < 1 || !face_off ||
      !faces || !vertices || !key || (num_samples > 0 && (!points || !face_choices)))
    return DIBR_B200_EINVAL;
  const dibr_layout::SamplePointsForwardLayout L = dibr_layout::sample_points_forward_layout(batch, total_faces);
  char* o = carve(workspace, workspace_bytes, L.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const Views m = views(batch, total_faces, num_vertices, fstride, vstride, face_off, faces);
  if (dtype == DIBR_B200_DTYPE_F32)
    return sample_forward<float>(m, num_samples, feature_dim, (const float*)vertices, areas, (const float*)face_features,
                                 key, (float*)points, face_choices, (float*)features, status, o, L, st);
  return sample_forward<double>(m, num_samples, feature_dim, (const double*)vertices, areas,
                                (const double*)face_features, key, (double*)points, face_choices, (double*)features,
                                status, o, L, st);
}

int dibr_b200_sample_points_backward(int batch, int64_t total_faces, int num_vertices, int64_t fstride,
                                     int64_t vstride, int dtype, int num_samples, int feature_dim,
                                     const int64_t* face_off, const int64_t* key, const int64_t* face_choices,
                                     const void* grad_points, const void* grad_features, const int32_t* corner_ptr,
                                     const int32_t* corners, void* grad_vertices, void* grad_face_features,
                                     void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream) {
  if (int r = check_dims(batch, total_faces, num_samples, dtype)) return r;
  const bool nv = grad_vertices != nullptr, nf = grad_face_features != nullptr;
  if (num_vertices < 0 || feature_dim < 0 || !workspace || batch < 1 || total_faces < 1 || !face_off || !key ||
      (num_samples > 0 && !face_choices) || (nv && (!grad_points || !corner_ptr || !corners)) ||
      (nf && (!grad_features || fstride == 0)))
    return DIBR_B200_EINVAL;
  const dibr_layout::SamplePointsBackwardLayout L =
      dibr_layout::sample_points_backward_layout(batch, total_faces, num_samples, tsize_of(dtype));
  char* o = carve(workspace, workspace_bytes, L.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  if (!nv && !nf) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const Views m = views(batch, total_faces, num_vertices, fstride, vstride, face_off, nullptr);
  if (dtype == DIBR_B200_DTYPE_F32)
    return sample_backward<float>(m, num_samples, feature_dim, key, face_choices, (const float*)grad_points,
                                  (const float*)grad_features, corner_ptr, corners, (float*)grad_vertices,
                                  (float*)grad_face_features, o, L, st);
  return sample_backward<double>(m, num_samples, feature_dim, key, face_choices, (const double*)grad_points,
                                 (const double*)grad_features, corner_ptr, corners, (double*)grad_vertices,
                                 (double*)grad_face_features, o, L, st);
}

}  // extern "C"
