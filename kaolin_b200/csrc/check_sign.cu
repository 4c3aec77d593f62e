// check_sign.cu — H100 implementation of Kaolin's point-in-mesh test (kaolin.ops.mesh.check_sign, CUDA path):
//   check_sign.py:45-57,138-155        per view: maxlen over all V vertices, verts and points / maxlen,
//                                      index_select of the corners, the operator below, count % 2 == 1
//   unbatched_mesh_intersection_cuda   kaolin/csrc/ops/mesh/mesh_intersection.cpp:32-65,
//                                      kernel mesh_intersection_cuda.cu:105-219
// behind the C ABI of include/dibr_b200.h.
//
// Semantics (reference kernel): a face (p1, p2, p3) counts for a point q when q's (y, z) lies in the face's
// CLOSED y-z box, taken with fminf/fmaxf (NaN skipped) and, in the double kernel, rounded to float
// (`float y_min = min(...)`); the signed volumes of q and q2 = (q.x + 10, q.y, q.z) against the face have
// different signs (> 0); the three direction-independent 2-D signed areas admit q; and the edge/vertex
// tie-break (:157-211, with the "completely vertical edge" rule) accepts it.  The reference tests every
// point against every face (O(N*F)), one float atomicAdd per hit.  Here:
//   * build (once per mesh, all views in one launch of each kernel): the per-view bounds and maxlen; one
//     pass over the faces that gathers and normalises the nine corner coordinates into one record and
//     stores the face's y-z box; the faces binned on a G x G y-z grid per view with DefTet's binning
//     (grid_bins.cuh, closed boxes), faces covering more than kMaxCells cells on the view's wide list.
//     An index outside [0, V) sets the status word (the reference's index_select faults on the device);
//   * query: the points of every view are counting-sorted by cell (count -> scan -> scatter of point
//     ids), so the threads of a warp walk the same face list; one thread per point tests its cell's faces
//     and the wide list, counts in an integer register and writes one byte, at the point's input index.
// Why the binning never drops a pair the reference counts: the cell function of grid_bins.cuh,
// clamp((int)((v - y0) * s), 0, G - 1) with a plain rounded subtraction and product, is monotone under
// round-to-nearest and clamps +-inf to the border cells.  A face's box bounds are floats; a point's
// coordinate is rounded to float for its cell (exact in the float kernel), and rounding is monotone, so
// whenever ymin <= q.y <= ymax (in the point's type) the point's cell lies within the face's cell range,
// on both axes.  Two input classes are not binned by that argument, and neither can count:
//   * a face whose box has an all-NaN component (all three corners NaN on that axis): its cross product
//     is NaN, so NaN > 0 is false for q and q2 alike and the signed-volume test fails; it is dropped;
//   * a point with a NaN coordinate: the same NaN reaches both signed volumes (x) or the cross product
//     (y, z); it takes cell 0 and is tested there, without a hit.
// Integer counts are exact and order-free, so equal predicates give equal outputs whatever the search
// structure.  The predicate follows the expression tree nvcc 12.9 generates for the reference's <float>
// and <double> instantiations (sm_90a, -O3), read from their SASS: 17 FFMA, 18 FMUL, 48 FADD in the float
// kernel and 17 DFMA, 18 DMUL, 48 DADD in the double kernel, with the same contraction in both:
//   cross(e, f)   x = fma(e.y, f.z, -(e.z * f.y)), y = fma(e.z, f.x, -(e.x * f.z)), z = fma(e.x, f.y, -(e.y * f.x))
//   dot(c, g)     fma(c.z, g.z, fma(c.x, g.x, c.y * g.y))
//   signed_area   fma(first difference product, (second difference product)), negated in the flipped branch
//   above_line    fma(r.x - l.x, v.y - l.y, -((r.y - l.y) * (v.x - l.x)))
// ("(...)" a rounded product; e = p1 - q, f = p2 - q, g = p3 - q, each component rounded).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dibr_b200.h"
#include "grid_bins.cuh"

namespace {

using dibr_layout::carve;
using dibr_layout::piece;

constexpr int kQueryThreads = 256;

// Correctly rounded operations, never contracted: the predicate spells out every FMA itself.
template <typename T> struct Rn;
template <> struct Rn<float> {
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float fma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
  static __device__ __forceinline__ float div(float a, float b) { return __fdiv_rn(a, b); }
  static __device__ __forceinline__ float to_float(float a) { return a; }
  static __device__ __forceinline__ float lo(float a, float b) { return fminf(a, b); }
  static __device__ __forceinline__ float hi(float a, float b) { return fmaxf(a, b); }
};
template <> struct Rn<double> {
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
  static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
  static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
  static __device__ __forceinline__ double fma(double a, double b, double c) { return __fma_rn(a, b, c); }
  static __device__ __forceinline__ double div(double a, double b) { return __ddiv_rn(a, b); }
  static __device__ __forceinline__ float to_float(double a) { return __double2float_rn(a); }
  static __device__ __forceinline__ double lo(double a, double b) { return fmin(a, b); }
  static __device__ __forceinline__ double hi(double a, double b) { return fmax(a, b); }
};

// torch.min / torch.max: NaN propagates
template <typename T> __device__ __forceinline__ T nan_min(T a, T b) { return (a < b || a != a) ? a : b; }
template <typename T> __device__ __forceinline__ T nan_max(T a, T b) { return (a > b || a != a) ? a : b; }

// Per view: maxlen = max over axes of (max - min) over all V vertices, NaN propagating (check_sign.py:
// 138-141: torch.max / torch.min / torch.max over the stacked lengths).
template <typename T>
__global__ void __launch_bounds__(1024) cs_maxlen_kernel(int V, const T* __restrict__ verts, T* __restrict__ maxlen) {
  const int b = blockIdx.x;
  const T* v = verts + (size_t)b * V * 3;
  T mn[3], mx[3];
  for (int k = 0; k < 3; ++k) { mn[k] = INFINITY; mx[k] = -INFINITY; }
  for (int i = threadIdx.x; i < V; i += blockDim.x)
    for (int k = 0; k < 3; ++k) {
      const T x = v[(size_t)i * 3 + k];
      mn[k] = nan_min(mn[k], x); mx[k] = nan_max(mx[k], x);
    }
  __shared__ T s[6][32];
  for (int d = 16; d > 0; d >>= 1)
    for (int k = 0; k < 3; ++k) {
      mn[k] = nan_min(mn[k], __shfl_xor_sync(kGridFull, mn[k], d));
      mx[k] = nan_max(mx[k], __shfl_xor_sync(kGridFull, mx[k], d));
    }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0)
    for (int k = 0; k < 3; ++k) { s[k][w] = mn[k]; s[3 + k][w] = mx[k]; }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i)
    for (int k = 0; k < 3; ++k) { mn[k] = nan_min(mn[k], s[k][i]); mx[k] = nan_max(mx[k], s[3 + k][i]); }
  T m = Rn<T>::sub(mx[0], mn[0]);
  for (int k = 1; k < 3; ++k) m = nan_max(m, Rn<T>::sub(mx[k], mn[k]));
  maxlen[b] = m;
}

// Per view: the grid over the y-z extent of the face boxes (NaN skipped).  Any finite grid keeps the
// binning exact; a tight one keeps the cell lists short.
__global__ void __launch_bounds__(1024) cs_grid_kernel(int F, int G, const float4* __restrict__ boxes,
                                                       float* __restrict__ bounds) {
  const int b = blockIdx.x;
  float lo0 = INFINITY, lo1 = INFINITY, hi0 = -INFINITY, hi1 = -INFINITY;
  for (int i = threadIdx.x; i < F; i += blockDim.x) {
    const float4 bb = boxes[(size_t)b * F + i];
    lo0 = fminf(lo0, bb.x); lo1 = fminf(lo1, bb.y); hi0 = fmaxf(hi0, bb.z); hi1 = fmaxf(hi1, bb.w);
  }
  __shared__ float s[4][32];
  for (int d = 16; d > 0; d >>= 1) {
    lo0 = fminf(lo0, __shfl_xor_sync(kGridFull, lo0, d)); lo1 = fminf(lo1, __shfl_xor_sync(kGridFull, lo1, d));
    hi0 = fmaxf(hi0, __shfl_xor_sync(kGridFull, hi0, d)); hi1 = fmaxf(hi1, __shfl_xor_sync(kGridFull, hi1, d));
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { s[0][w] = lo0; s[1][w] = lo1; s[2][w] = hi0; s[3][w] = hi1; }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) {
    lo0 = fminf(lo0, s[0][i]); lo1 = fminf(lo1, s[1][i]); hi0 = fmaxf(hi0, s[2][i]); hi1 = fmaxf(hi1, s[3][i]);
  }
  const float lo[2] = {lo0, lo1}, hi[2] = {hi0, hi1};
  float* o = bounds + 4 * b;
  for (int k = 0; k < 2; ++k) {
    float a = lo[k], z = hi[k];
    if (!(z >= a) || !(z - a < INFINITY)) { a = 0.f; z = 1.f; }   // no finite extent (or no face)
    o[k] = a;
    o[2 + k] = (float)G / fmaxf(z - a, 1e-20f);
  }
}

// One record of nine normalised corner coordinates and one float y-z box {ymin, zmin, ymax, zmax} per
// (view, face).  With faces: the corners are verts[b][faces[f][k]] / maxlen[b] (index_select of the
// divided vertices); without: they are v1, v2, v3 [f] as given (the raw operator, one view).
template <typename T>
__global__ void __launch_bounds__(256) cs_faces_kernel(int B, int V, int F, const T* __restrict__ verts,
                                                       const int64_t* __restrict__ faces, const T* __restrict__ maxlen,
                                                       const T* __restrict__ v1, const T* __restrict__ v2,
                                                       const T* __restrict__ v3, T* __restrict__ records,
                                                       float4* __restrict__ boxes, int* __restrict__ status) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * F) return;
  const int b = (int)(i / F), f = (int)(i - (int64_t)b * F);
  T p[9];
  if (faces) {
    const T m = maxlen[b];
    for (int k = 0; k < 3; ++k) {
      const int64_t vi = faces[(size_t)f * 3 + k];
      if (vi < 0 || vi >= V) { atomicOr(status, 1); return; }
      const T* src = verts + ((size_t)b * V + vi) * 3;
      for (int c = 0; c < 3; ++c) p[k * 3 + c] = Rn<T>::div(src[c], m);
    }
  } else {
    for (int c = 0; c < 3; ++c) { p[c] = v1[(size_t)f * 3 + c]; p[3 + c] = v2[(size_t)f * 3 + c]; p[6 + c] = v3[(size_t)f * 3 + c]; }
  }
  T* r = records + i * 9;
  for (int k = 0; k < 9; ++k) r[k] = p[k];
  // mesh_intersection_cuda.cu:51-54: float y_min = min(b.y, min(c.y, d.y)), ...
  boxes[i] = make_float4(Rn<T>::to_float(Rn<T>::lo(p[1], Rn<T>::lo(p[4], p[7]))),
                         Rn<T>::to_float(Rn<T>::lo(p[2], Rn<T>::lo(p[5], p[8]))),
                         Rn<T>::to_float(Rn<T>::hi(p[1], Rn<T>::hi(p[4], p[7]))),
                         Rn<T>::to_float(Rn<T>::hi(p[2], Rn<T>::hi(p[5], p[8]))));
}

template <typename T>
__device__ __forceinline__ void load_point(const T* __restrict__ points, const T* __restrict__ maxlen, int b, int64_t i,
                                           T& x, T& y, T& z) {
  const T* q = points + i * 3;
  x = q[0]; y = q[1]; z = q[2];
  if (maxlen) { const T m = maxlen[b]; x = Rn<T>::div(x, m); y = Rn<T>::div(y, m); z = Rn<T>::div(z, m); }
}

// Query, step 1: every point's cell, and the per-cell point counts.
template <typename T>
__global__ void __launch_bounds__(256) cs_point_cell_kernel(Grid pg, const T* __restrict__ points,
                                                            const T* __restrict__ maxlen, int* __restrict__ pcell) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)pg.B * pg.P) return;
  const int b = (int)(i / pg.P);
  T x, y, z;
  load_point(points, maxlen, b, i, x, y, z);
  const float* bd = pg.bounds + 4 * b;
  const int c = cell_of(Rn<T>::to_float(z), bd[1], bd[3], pg.G) * pg.G + cell_of(Rn<T>::to_float(y), bd[0], bd[2], pg.G);
  pcell[i] = c;
  atomicAdd(pg.cnt + (size_t)b * (pg.G * pg.G + 1) + c, 1);
}

// Query, step 3 (after grid_scan_kernel over the point counts): the point ids, grouped by cell.
__global__ void __launch_bounds__(256) cs_point_scatter_kernel(Grid pg, const int* __restrict__ pcell,
                                                               int* __restrict__ order) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)pg.B * pg.P) return;
  const int b = (int)(i / pg.P);
  const size_t row = (size_t)b * (pg.G * pg.G + 1) + pcell[i];
  const int pos = pg.off[row] + atomicAdd(pg.cnt + row, 1);
  order[(size_t)b * pg.P + pos] = (int)(i - (int64_t)b * pg.P);
}

template <typename T> struct P2 { T x, y; };   // (y, z) of a 3-D point, the reference's vec2 view

// mesh_intersection_cuda.cu:69-83
template <typename T>
__device__ __forceinline__ T signed_area(P2<T> a, P2<T> b, P2<T> c) {
  using R = Rn<T>;
  if (c.x > b.x || (b.x == c.x && c.y < b.y))
    return -R::fma(R::sub(b.y, c.y), R::sub(a.x, c.x), R::mul(R::sub(c.x, b.x), R::sub(a.y, c.y)));
  return R::fma(R::sub(c.y, b.y), R::sub(a.x, b.x), R::mul(R::sub(b.x, c.x), R::sub(a.y, b.y)));
}

// mesh_intersection_cuda.cu:85-93
template <typename T>
__device__ __forceinline__ bool above_line(P2<T> v, P2<T> l, P2<T> r) {
  using R = Rn<T>;
  return R::fma(R::sub(r.x, l.x), R::sub(v.y, l.y), -R::mul(R::sub(r.y, l.y), R::sub(v.x, l.x))) > T(0);
}

// mesh_intersection_cuda.cu:131-214 for one (point, face); q2x = q.x + 10.
template <typename T>
__device__ __forceinline__ bool crosses(const T* __restrict__ rec, float4 box, T qx, T qy, T qz, T q2x) {
  using R = Rn<T>;
  if (qy < (T)box.x || (T)box.z < qy || qz < (T)box.y || (T)box.w < qz) return false;
  const T p1x = rec[0], p1y = rec[1], p1z = rec[2], p2x = rec[3], p2y = rec[4], p2z = rec[5];
  const T p3x = rec[6], p3y = rec[7], p3z = rec[8];
  // signed_volume(q, p1, p2, p3) = dot(cross(p1 - q, p2 - q), p3 - q), and the same for q2
  const T ex = R::sub(p1x, qx), ey = R::sub(p1y, qy), ez = R::sub(p1z, qz);
  const T fx = R::sub(p2x, qx), fy = R::sub(p2y, qy), fz = R::sub(p2z, qz);
  const T gx = R::sub(p3x, qx), gy = R::sub(p3y, qy), gz = R::sub(p3z, qz);
  const T ex2 = R::sub(p1x, q2x), fx2 = R::sub(p2x, q2x), gx2 = R::sub(p3x, q2x);
  const T cx = R::fma(ey, fz, -R::mul(ez, fy));
  const T cy = R::fma(ez, fx, -R::mul(ex, fz)), cz = R::fma(ex, fy, -R::mul(ey, fx));
  const T cy2 = R::fma(ez, fx2, -R::mul(ex2, fz)), cz2 = R::fma(ex2, fy, -R::mul(ey, fx2));
  const T vol1 = R::fma(cz, gz, R::fma(cx, gx, R::mul(cy, gy)));
  const T vol2 = R::fma(cz2, gz, R::fma(cx, gx2, R::mul(cy2, gy)));
  if ((vol1 > T(0)) == (vol2 > T(0))) return false;
  const P2<T> q{qy, qz}, a{p1y, p1z}, b{p2y, p2z}, c{p3y, p3z};
  const T d1 = signed_area(q, a, b), d2 = signed_area(q, b, c);
  if (!(R::mul(d1, d2) >= T(0))) return false;
  const T d3 = signed_area(q, c, a);
  if (!(R::mul(d3, d1) >= T(0) && R::mul(d2, d3) >= T(0))) return false;
  bool edge;
  P2<T> v1, v2, other;
  if (q.x == a.x && q.y == a.y)      { edge = false; v1 = b; v2 = c; }
  else if (q.x == b.x && q.y == b.y) { edge = false; v1 = a; v2 = c; }
  else if (q.x == c.x && q.y == c.y) { edge = false; v1 = a; v2 = b; }
  else if (d1 == T(0))               { edge = true; v1 = a; v2 = b; other = c; }
  else if (d2 == T(0))               { edge = true; v1 = b; v2 = c; other = a; }
  else if (d3 == T(0))               { edge = true; v1 = c; v2 = a; other = b; }
  else return true;
  if (v1.x > v2.x || (v1.x == v2.x && v1.y > v2.y)) { const P2<T> t = v1; v1 = v2; v2 = t; }
  // count only the face "below" the point; for a completely vertical edge, the one to its left
  if (edge) return !above_line(other, v1, v2);
  return above_line(q, v1, v2) && v1.x < q.x && v2.x >= q.x;
}

template <typename T>
struct QueryArgs {
  Grid g;                      // the build's face grid
  const int* pcell; const int* order;
  const T* points; const T* maxlen; const T* records; const float4* boxes;
  uint8_t* inside;             // (B, N) parity, or NULL
  T* counts;                   // (B, N) counts, or NULL
};

// Query, step 4: one thread per point, in cell order; the output goes to the point's input index.
template <typename T>
__global__ void __launch_bounds__(kQueryThreads) cs_query_kernel(const __grid_constant__ QueryArgs<T> a) {
  const Grid& g = a.g;
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= (int64_t)g.B * g.P) return;
  const int b = (int)(s / g.P);
  const int64_t i = (int64_t)b * g.P + __ldg(a.order + s);
  T qx, qy, qz;
  load_point(a.points, a.maxlen, b, i, qx, qy, qz);
  const T q2x = Rn<T>::add(qx, T(10));
  const int ncell = g.G * g.G, cell = __ldg(a.pcell + i);
  const int* cnt = g.cnt + (size_t)b * (ncell + 1);
  const int* off = g.off + (size_t)b * (ncell + 1);
  const int64_t fbase = (int64_t)b * g.F;
  int n = 0;
  auto visit = [&](const int* list, int len) {
    for (int k = 0; k < len; ++k) {
      const int64_t face = fbase + __ldg(list + k);
      n += crosses(a.records + face * 9, __ldg(a.boxes + face), qx, qy, qz, q2x) ? 1 : 0;
    }
  };
  visit(g.entries + (size_t)b * g.F * kMaxCells + off[cell], cnt[cell]);
  visit(g.wide + (size_t)b * g.F, off[ncell]);
  if (a.inside) a.inside[i] = (uint8_t)(n & 1);
  if (a.counts) a.counts[i] = (T)n;
}

struct Mesh {   // the build workspace carved
  Grid g;
  void* counters; size_t counters_bytes;   // the grid's cnt and off
  void* maxlen; void* records; float4* boxes;
};

int carve_build(int B, int F, size_t tsize, void* ws, size_t bytes, Mesh& m) {
  const dibr_layout::CheckSignBuildLayout L = dibr_layout::check_sign_build_layout(B, F, tsize);
  char* o = carve(ws, bytes, L.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  m.g.B = B; m.g.F = F; m.g.P = 0; m.g.G = grid_side(F);
  m.g.bounds = piece<float>(o, L.grid.bounds);
  m.g.cnt = piece<int>(o, L.grid.cnt);
  m.g.off = piece<int>(o, L.grid.off);
  m.g.entries = piece<int>(o, L.grid.entries);
  m.g.wide = piece<int>(o, L.grid.wide);
  m.counters = piece<char>(o, L.grid.counters);
  m.counters_bytes = L.grid.counters.bytes;
  m.maxlen = piece<char>(o, L.maxlen);
  m.boxes = piece<float4>(o, L.boxes);
  m.records = piece<char>(o, L.records);
  return 0;
}

int check_sizes(int B, int F, int N) {
  if ((int64_t)B * F * kMaxCells >= 0x7fffffffLL || (int64_t)B * N >= 0x7fffffffLL) return DIBR_B200_ESIZE;
  return 0;
}

unsigned blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

// verts/faces (build) or v1/v2/v3 (raw, maxlen not used)
template <typename T>
int build(int B, int V, int F, const T* verts, const int64_t* faces, const T* v1, const T* v2, const T* v3,
          int32_t* status, const Mesh& m, cudaStream_t st) {
  Grid g = m.g;
  cudaError_t e = cudaMemsetAsync(m.counters, 0, m.counters_bytes, st);
  if (e != cudaSuccess) return (int)e;
  if (status) {
    e = cudaMemsetAsync(status, 0, sizeof(int32_t), st);
    if (e != cudaSuccess) return (int)e;
  }
  T* maxlen = (T*)m.maxlen;
  if (!v1) cs_maxlen_kernel<T><<<B, 1024, 0, st>>>(V, verts, maxlen);   // the gather path normalises
  const int64_t nf = (int64_t)B * F;
  if (nf > 0)
    cs_faces_kernel<T><<<blocks(nf, 256), 256, 0, st>>>(B, V, F, verts, faces, maxlen, v1, v2, v3, (T*)m.records,
                                                         m.boxes, status);
  cs_grid_kernel<<<B, 1024, 0, st>>>(F, g.G, m.boxes, const_cast<float*>(g.bounds));
  if (nf == 0) return (int)cudaGetLastError();
  grid_bin_kernel<true, false><<<blocks(nf, 256), 256, 0, st>>>(g, (const float*)m.boxes);
  grid_scan_kernel<<<B, 1024, 0, st>>>(g);
  grid_bin_kernel<true, true><<<blocks(nf, 256), 256, 0, st>>>(g, (const float*)m.boxes);
  return (int)cudaGetLastError();
}

template <typename T>
int query(int N, const T* points, const T* maxlen, const Mesh& m, uint8_t* inside, T* counts, void* ws, size_t bytes,
          cudaStream_t st) {
  const int B = m.g.B, F = m.g.F;
  const dibr_layout::CheckSignQueryLayout L = dibr_layout::check_sign_query_layout(B, F, N);
  char* o = carve(ws, bytes, L.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  if (N == 0) return 0;
  Grid pg = m.g;          // the same cells, counting points
  pg.P = N;
  pg.cnt = piece<int>(o, L.cnt);
  pg.off = piece<int>(o, L.off);
  int* pcell = piece<int>(o, L.pcell);
  int* order = piece<int>(o, L.order);
  cudaError_t e = cudaMemsetAsync(pg.cnt, 0, L.cnt.bytes, st);
  if (e != cudaSuccess) return (int)e;
  const int64_t np = (int64_t)B * N;
  cs_point_cell_kernel<T><<<blocks(np, 256), 256, 0, st>>>(pg, points, maxlen, pcell);
  grid_scan_kernel<<<B, 1024, 0, st>>>(pg);
  cs_point_scatter_kernel<<<blocks(np, 256), 256, 0, st>>>(pg, pcell, order);
  QueryArgs<T> a;
  a.g = m.g; a.g.P = N;
  a.pcell = pcell; a.order = order; a.points = points; a.maxlen = maxlen;
  a.records = (const T*)m.records; a.boxes = m.boxes; a.inside = inside; a.counts = counts;
  cs_query_kernel<T><<<blocks(np, kQueryThreads), kQueryThreads, 0, st>>>(a);
  return (int)cudaGetLastError();
}

size_t tsize_of(int dtype) {
  return dtype == DIBR_B200_DTYPE_F32 ? sizeof(float) : dtype == DIBR_B200_DTYPE_F64 ? sizeof(double) : 0;
}

}  // namespace

extern "C" {

int dibr_b200_check_sign_workspace_bytes(int batch, int num_faces, int num_points, int dtype, size_t* build_bytes,
                                         size_t* query_bytes) {
  const size_t ts = tsize_of(dtype);
  if (batch <= 0 || num_faces < 0 || num_points < 0 || ts == 0) return DIBR_B200_EINVAL;
  if (int r = check_sizes(batch, num_faces, num_points)) return r;
  if (build_bytes) *build_bytes = dibr_layout::check_sign_build_layout(batch, num_faces, ts).bytes;
  if (query_bytes) *query_bytes = dibr_layout::check_sign_query_layout(batch, num_faces, num_points).bytes;
  return 0;
}

int dibr_b200_check_sign_build(int batch, int num_vertices, int num_faces, int dtype, const void* verts,
                               const int64_t* faces, int32_t* status, void* workspace, size_t workspace_bytes,
                               dibr_b200_stream_t stream) {
  const size_t ts = tsize_of(dtype);
  if (batch <= 0 || num_vertices < 0 || num_faces < 0 || ts == 0) return DIBR_B200_EINVAL;
  if (!status || !workspace || (num_vertices > 0 && !verts) || (num_faces > 0 && !faces)) return DIBR_B200_EINVAL;
  if (int r = check_sizes(batch, num_faces, 0)) return r;
  Mesh m;
  if (int r = carve_build(batch, num_faces, ts, workspace, workspace_bytes, m)) return r;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == DIBR_B200_DTYPE_F32)
    return build<float>(batch, num_vertices, num_faces, (const float*)verts, faces, nullptr, nullptr, nullptr, status, m, st);
  return build<double>(batch, num_vertices, num_faces, (const double*)verts, faces, nullptr, nullptr, nullptr, status, m,
                       st);
}

int dibr_b200_check_sign_query(int batch, int num_faces, int num_points, int dtype, const void* points,
                               const void* mesh, size_t mesh_bytes, uint8_t* inside, void* workspace,
                               size_t workspace_bytes, dibr_b200_stream_t stream) {
  const size_t ts = tsize_of(dtype);
  if (batch <= 0 || num_faces < 0 || num_points < 0 || ts == 0) return DIBR_B200_EINVAL;
  if (!mesh || !workspace || (num_points > 0 && (!points || !inside))) return DIBR_B200_EINVAL;
  if (int r = check_sizes(batch, num_faces, num_points)) return r;
  Mesh m;
  if (int r = carve_build(batch, num_faces, ts, const_cast<void*>(mesh), mesh_bytes, m)) return r;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == DIBR_B200_DTYPE_F32)
    return query<float>(num_points, (const float*)points, (const float*)m.maxlen, m, inside, nullptr, workspace,
                        workspace_bytes, st);
  return query<double>(num_points, (const double*)points, (const double*)m.maxlen, m, inside, nullptr, workspace,
                       workspace_bytes, st);
}

int dibr_b200_mesh_intersection_count(int num_faces, int num_points, int dtype, const void* points, const void* verts_1,
                                      const void* verts_2, const void* verts_3, void* counts, void* workspace,
                                      size_t workspace_bytes, dibr_b200_stream_t stream) {
  const size_t ts = tsize_of(dtype);
  if (num_faces < 0 || num_points < 0 || ts == 0 || !workspace) return DIBR_B200_EINVAL;
  if (num_points > 0 && (!points || !counts)) return DIBR_B200_EINVAL;
  if (num_faces > 0 && (!verts_1 || !verts_2 || !verts_3)) return DIBR_B200_EINVAL;
  if (int r = check_sizes(1, num_faces, num_points)) return r;
  const size_t nb = dibr_layout::check_sign_build_layout(1, num_faces, ts).bytes;
  if (workspace_bytes < nb + dibr_layout::check_sign_query_layout(1, num_faces, num_points).bytes)
    return DIBR_B200_EWORKSPACE;
  Mesh m;
  if (int r = carve_build(1, num_faces, ts, workspace, nb, m)) return r;
  cudaStream_t st = (cudaStream_t)stream;
  void* qws = (char*)workspace + nb;
  const size_t qbytes = workspace_bytes - nb;
  if (dtype == DIBR_B200_DTYPE_F32) {
    int r = build<float>(1, 0, num_faces, nullptr, nullptr, (const float*)verts_1, (const float*)verts_2,
                         (const float*)verts_3, nullptr, m, st);
    return r ? r : query<float>(num_points, (const float*)points, nullptr, m, nullptr, (float*)counts, qws, qbytes, st);
  }
  int r = build<double>(1, 0, num_faces, nullptr, nullptr, (const double*)verts_1, (const double*)verts_2,
                        (const double*)verts_3, nullptr, m, st);
  return r ? r : query<double>(num_points, (const double*)points, nullptr, m, nullptr, (double*)counts, qws, qbytes, st);
}

}  // extern "C"
