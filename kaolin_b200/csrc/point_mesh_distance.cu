// point_mesh_distance.cu — H100 implementation of Kaolin's point-to-mesh distance
// (kaolin.metrics.trianglemesh.point_to_mesh_distance, CUDA path):
//   trianglemesh.py:87-99                 per view: the operator below, then torch.stack of the outputs
//   unbatched_triangle_distance_*_cuda    kaolin/csrc/metrics/unbatched_triangle_distance.cpp,
//                                         kernels unbatched_triangle_distance_cuda.cu:177-416
// behind the C ABI of include/dibr_b200.h.
//
// Exact by construction: every (point, face) pair is evaluated, as the reference does; all views go
// through one launch of each kernel and no call reads anything back to the host.
//   forward   pmd_faces_kernel     one record per (view, face) of every per-face value the reference
//                                  recomputes for each pair (edges, squared lengths, edge normals, unit
//                                  normal), each by the reference's own operations;
//             pmd_search_kernel    CTAs over (view, point block, face chunk); a chunk's records are staged
//                                  in shared memory, each thread keeps kPointsPerThread points and, per
//                                  point, the 64-bit key (dist_bits << 32) | face of its best pair, merged
//                                  into the point's key with atomicMin.  dist is a non-negative float or
//                                  NaN in both dtypes (the double kernel also narrows it to float), NaN
//                                  maps to 0xFFFFFFFF, so the smallest key is the smallest distance and,
//                                  among equals, the lowest face index: the reference's tie rule.  The
//                                  atomics' order cannot change the minimum;
//             pmd_finalize_kernel  decodes the winning face and re-evaluates that pair with its type.
//   backward  pmd_point_grad_kernel  the reference's per-type expressions (grad_out = 2 * grad_dist),
//                                  grad_points and the point's face terms; then the points are grouped by
//                                  (view, closest face): count -> exclusive scan -> atomic-cursor fill ->
//                                  per-row ascending sort (row_sort.cuh), and pmd_face_grad_kernel adds each
//                                  face's terms in ascending point order onto grad_face_vertices.  No float
//                                  atomics: the face gradients are deterministic.
//
// Deliberate deviation: a pair whose distance is NaN never wins unless every face of the point is NaN,
// and then face 0 wins (its distance and type are written).  The reference seeds each 512-face tile's
// minimum with the tile's first face, so a NaN face at an index that is a multiple of 512 discards the
// rest of its tile (and at index 0 makes the point's result NaN).
//
// Rounding follows the expression tree nvcc 12.9 generates for the reference's <float, float3> and
// <double, double3> kernels (sm_90a, -O3), read from their PTX and SASS; the same contraction in both
// dtypes (a rounded product written (...)):
//   dot(a, b)         fma(a.z, b.z, fma(a.x, b.x, (a.y * b.y)))
//   cross(a, b)       x = fma(a.y, b.z, -(a.z * b.y)), y = fma(a.z, b.x, -(a.x * b.z)), z = fma(a.x, b.y, -(a.y * b.x))
//   point_at(v, e, t) fma(e, t, v), t narrowed to float in the double kernel
//   project_plane     fma(-unit_normal, dot(p - v1, unit_normal), p); unit_normal = normal * rsqrt(dot(normal, normal))
//   divisions IEEE (never a reciprocal multiply), 1 / m a correctly rounded reciprocal, sqrt correctly rounded;
//   clamp(k, 0, 1) of the float backward a saturating add (FADD.SAT), of the double one fmax(0, fmin(1, k));
//   the reference's float atomicAdd is an FTZ add, so the float face gradients are summed with add.rn.ftz.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dibr_b200.h"
#include "op_layouts.h"
#include "row_sort.cuh"
#include "scan.cuh"

namespace {

using dibr_b200_detail::exclusive_scan;
using dibr_layout::carve;
using dibr_layout::kFaceRecord;
using dibr_layout::piece;

constexpr int kThreads = 256;
constexpr int kSearchThreads = 128;
constexpr int kPointsPerThread = 4;
constexpr int kSearchPoints = kSearchThreads * kPointsPerThread;   // points per CTA
constexpr int kTileFaces = 64;          // face records staged in shared memory at a time
constexpr int kCtasPerSm = 8;           // search CTAs aimed at per SM when choosing the face chunks
constexpr int kShortRow = 32;           // rows of at most this many points are sorted by one thread
constexpr int kLongCtas = 132;          // CTAs that share out the long rows
constexpr int kSortThreads = 1024;

// Record offsets (kFaceRecord values of T per face).
enum { R_V1 = 0, R_V2 = 3, R_V3 = 6, R_E12 = 9, R_E23 = 12, R_E31 = 15, R_N12 = 18, R_N23 = 21, R_N31 = 24,
       R_UN = 27, R_L12 = 30, R_L23 = 31, R_L31 = 32 };
static_assert(kFaceRecord == 33, "record layout");

// Correctly rounded operations, never contracted: every FMA is spelled out.
template <typename T> struct Rn;
template <> struct Rn<float> {
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float fma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
  static __device__ __forceinline__ float div(float a, float b) { return __fdiv_rn(a, b); }
  static __device__ __forceinline__ float rcp(float a) { return __frcp_rn(a); }
  static __device__ __forceinline__ float sqrt(float a) { return __fsqrt_rn(a); }
  static __device__ __forceinline__ float rsqrt(float a) { return rsqrtf(a); }
  static __device__ __forceinline__ float narrow(float a) { return a; }
  static __device__ __forceinline__ float clamp01(float a) {
    float r;
    asm("add.sat.f32 %0, 0f00000000, %1;" : "=f"(r) : "f"(a));
    return r;
  }
  // the reference's atomicAdd(float): RED.ADD.F32.FTZ.RN
  static __device__ __forceinline__ float acc(float a, float b) {
    float r;
    asm("add.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
  }
};
template <> struct Rn<double> {
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
  static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
  static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
  static __device__ __forceinline__ double fma(double a, double b, double c) { return __fma_rn(a, b, c); }
  static __device__ __forceinline__ double div(double a, double b) { return __ddiv_rn(a, b); }
  static __device__ __forceinline__ double rcp(double a) { return __drcp_rn(a); }
  static __device__ __forceinline__ double sqrt(double a) { return __dsqrt_rn(a); }
  static __device__ __forceinline__ double rsqrt(double a) { return ::rsqrt(a); }
  static __device__ __forceinline__ float narrow(double a) { return __double2float_rn(a); }
  static __device__ __forceinline__ double clamp01(double a) { return fmax(0.0, fmin(1.0, a)); }
  static __device__ __forceinline__ double acc(double a, double b) { return __dadd_rn(a, b); }
};

template <typename T> struct V3 { T x, y, z; };

template <typename T> __device__ __forceinline__ V3<T> ld3(const T* p) { return {p[0], p[1], p[2]}; }
template <typename T> __device__ __forceinline__ void st3(T* p, V3<T> v) { p[0] = v.x; p[1] = v.y; p[2] = v.z; }

template <typename T> __device__ __forceinline__ V3<T> sub(V3<T> a, V3<T> b) {
  return {Rn<T>::sub(a.x, b.x), Rn<T>::sub(a.y, b.y), Rn<T>::sub(a.z, b.z)};
}
template <typename T> __device__ __forceinline__ V3<T> add(V3<T> a, V3<T> b) {
  return {Rn<T>::add(a.x, b.x), Rn<T>::add(a.y, b.y), Rn<T>::add(a.z, b.z)};
}
template <typename T> __device__ __forceinline__ V3<T> scale(V3<T> a, T s) {
  return {Rn<T>::mul(a.x, s), Rn<T>::mul(a.y, s), Rn<T>::mul(a.z, s)};
}
template <typename T> __device__ __forceinline__ V3<T> neg(V3<T> a) { return {-a.x, -a.y, -a.z}; }
template <typename T> __device__ __forceinline__ T dot(V3<T> a, V3<T> b) {
  using R = Rn<T>;
  return R::fma(a.z, b.z, R::fma(a.x, b.x, R::mul(a.y, b.y)));
}
template <typename T> __device__ __forceinline__ V3<T> cross(V3<T> a, V3<T> b) {
  using R = Rn<T>;
  return {R::fma(a.y, b.z, -R::mul(a.z, b.y)), R::fma(a.z, b.x, -R::mul(a.x, b.z)),
          R::fma(a.x, b.y, -R::mul(a.y, b.x))};
}
// fma(a, s, c) per component
template <typename T> __device__ __forceinline__ V3<T> fma3(V3<T> a, T s, V3<T> c) {
  using R = Rn<T>;
  return {R::fma(a.x, s, c.x), R::fma(a.y, s, c.y), R::fma(a.z, s, c.z)};
}

// ---------------------------------------------------------------------------------------------
// Forward.

// One record per (view, face): unbatched_triangle_distance_cuda.cu:268-271 and the per-face parts of
// project_edge, is_not_above and project_plane (:133-168).
template <typename T>
__global__ void __launch_bounds__(kThreads) pmd_faces_kernel(int64_t nf, const T* __restrict__ fv, T* __restrict__ rec) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nf) return;
  const T* v = fv + i * 9;
  const V3<T> v1 = ld3(v), v2 = ld3(v + 3), v3 = ld3(v + 6);
  const V3<T> e12 = sub(v2, v1), e23 = sub(v3, v2), e31 = sub(v1, v3);
  const V3<T> normal = cross(sub(v1, v2), e31);
  const V3<T> unit = scale(normal, Rn<T>::rsqrt(dot(normal, normal)));
  T* r = rec + i * kFaceRecord;
  st3(r + R_V1, v1); st3(r + R_V2, v2); st3(r + R_V3, v3);
  st3(r + R_E12, e12); st3(r + R_E23, e23); st3(r + R_E31, e31);
  st3(r + R_N12, cross(normal, e12)); st3(r + R_N23, cross(normal, e23)); st3(r + R_N31, cross(normal, e31));
  st3(r + R_UN, unit);
  r[R_L12] = dot(e12, e12); r[R_L23] = dot(e23, e23); r[R_L31] = dot(e31, e31);
}

template <typename T> __device__ __forceinline__ bool in_range(T a) { return a <= T(1) && a >= T(0); }

// The squared distance of p to the face of record r, as the reference's forward computes it
// (:264-302), and its type when TYPE.
template <typename T, bool TYPE>
__device__ __forceinline__ float pair_distance(const T* r, V3<T> p, int* type) {
  using R = Rn<T>;
  const V3<T> v1 = ld3(r + R_V1), e12 = ld3(r + R_E12), v3 = ld3(r + R_V3), e31 = ld3(r + R_E31);
  const V3<T> pv1 = sub(p, v1), pv3 = sub(p, v3);
  const T uab = R::div(dot(pv1, e12), r[R_L12]);
  const T uca = R::div(dot(pv3, e31), r[R_L31]);
  V3<T> c;
  int t;
  if (uca > T(1) && uab < T(0)) {
    c = v1; t = 1;
  } else {
    const V3<T> v2 = ld3(r + R_V2), e23 = ld3(r + R_E23);
    const V3<T> pv2 = sub(p, v2);
    const T ubc = R::div(dot(pv2, e23), r[R_L23]);
    if (uab > T(1) && ubc < T(0)) {
      c = v2; t = 2;
    } else if (ubc > T(1) && uca < T(0)) {
      c = v3; t = 3;
    } else if (in_range(uab) && dot(ld3(r + R_N12), pv1) <= T(0)) {
      c = fma3(e12, (T)(float)uab, v1); t = 4;
    } else if (in_range(ubc) && dot(ld3(r + R_N23), pv2) <= T(0)) {
      c = fma3(e23, (T)(float)ubc, v2); t = 5;
    } else if (in_range(uca) && dot(ld3(r + R_N31), pv3) <= T(0)) {
      c = fma3(e31, (T)(float)uca, v3); t = 6;
    } else {
      const V3<T> un = ld3(r + R_UN);
      c = fma3(neg(un), dot(pv1, un), p); t = 0;
    }
  }
  if (TYPE) *type = t;
  const V3<T> d = sub(p, c);
  return R::narrow(dot(d, d));
}

__device__ __forceinline__ unsigned long long make_key(float d, int face) {
  const unsigned bits = d != d ? 0xFFFFFFFFu : __float_as_uint(d);
  return ((unsigned long long)bits << 32) | (unsigned)face;
}

// CTA c: view c / (PB * C), point block (c / C) % PB, face chunk c % C of `chunk` faces.
template <typename T>
__global__ void __launch_bounds__(kSearchThreads) pmd_search_kernel(int N, int F, int PB, int C, int chunk,
                                                                    const T* __restrict__ points,
                                                                    const T* __restrict__ rec,
                                                                    unsigned long long* __restrict__ keys) {
  __shared__ T s[kTileFaces * kFaceRecord];
  const int64_t c = blockIdx.x;
  const int fc = (int)(c % C);
  const int64_t rest = c / C;
  const int pb = (int)(rest % PB), b = (int)(rest / PB);
  const int f0 = fc * chunk, f1 = min(F, f0 + chunk);
  V3<T> p[kPointsPerThread];
  unsigned long long best[kPointsPerThread];
#pragma unroll
  for (int k = 0; k < kPointsPerThread; ++k) {
    const int n = pb * kSearchPoints + k * kSearchThreads + threadIdx.x;
    best[k] = ~0ull;
    p[k] = n < N ? ld3(points + ((int64_t)b * N + n) * 3) : V3<T>{T(0), T(0), T(0)};
  }
  const T* vrec = rec + (int64_t)b * F * kFaceRecord;
  for (int t0 = f0; t0 < f1; t0 += kTileFaces) {
    const int nt = min(kTileFaces, f1 - t0);
    __syncthreads();
    for (int j = threadIdx.x; j < nt * kFaceRecord; j += kSearchThreads) s[j] = vrec[(int64_t)t0 * kFaceRecord + j];
    __syncthreads();
    for (int j = 0; j < nt; ++j) {
      const T* r = s + j * kFaceRecord;
#pragma unroll
      for (int k = 0; k < kPointsPerThread; ++k) {
        const unsigned long long key = make_key(pair_distance<T, false>(r, p[k], nullptr), t0 + j);
        best[k] = key < best[k] ? key : best[k];
      }
    }
  }
#pragma unroll
  for (int k = 0; k < kPointsPerThread; ++k) {
    const int n = pb * kSearchPoints + k * kSearchThreads + threadIdx.x;
    if (n < N && f0 < f1) atomicMin(keys + (int64_t)b * N + n, best[k]);
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) pmd_finalize_kernel(int N, int F, const T* __restrict__ points,
                                                                const T* __restrict__ rec,
                                                                const unsigned long long* __restrict__ keys,
                                                                T* __restrict__ dist, int64_t* __restrict__ face_idx,
                                                                int32_t* __restrict__ dist_type, int64_t np) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= np) return;
  const int64_t b = i / N;
  const int face = (int)(keys[i] & 0xFFFFFFFFull);
  int t;
  const float d = pair_distance<T, true>(rec + (b * F + face) * kFaceRecord, ld3(points + i * 3), &t);
  dist[i] = (T)d;
  face_idx[i] = face;
  dist_type[i] = t;
}

// ---------------------------------------------------------------------------------------------
// Backward.

// The vertices (bit 0: v1, 1: v2, 2: v3) whose face gradient a point of type t adds to; any type other
// than 0-5 takes the reference's last branch, the edge e31.
__device__ __forceinline__ int touched(int t) {
  switch (t) {
    case 0: return 7;
    case 1: return 1;
    case 2: return 2;
    case 3: return 4;
    case 4: return 3;
    case 5: return 6;
    default: return 5;
  }
}

// compute_edge_backward (:177-233): the gradients of the point (pbar) and of the edge's ends va, vb.
template <typename T>
__device__ __forceinline__ void edge_backward(V3<T> vab, V3<T> pb, T grad, V3<T>& pbar, V3<T>& va, V3<T>& vb) {
  using R = Rn<T>;
  const T l = dot(pb, vab), m = dot(vab, vab);
  const T k = R::div(l, m);
  const T j = R::clamp01(k);
  const V3<T> i = fma3(vab, j, neg(pb));
  const V3<T> ibar = {R::mul(grad, i.x), R::mul(grad, i.y), R::mul(grad, i.z)};
  const T jbar = dot(ibar, vab);
  const T djdk = (k > T(0) && k < T(1)) ? T(1) : T(0);
  const T kbar = R::mul(jbar, djdk);
  const T mbar = R::mul(R::div(-l, R::mul(m, m)), kbar);
  const T lbar = R::mul(R::rcp(m), kbar);
  pbar = fma3(vab, lbar, neg(ibar));
  const V3<T> vab2 = add(vab, vab);
  const V3<T> inner = fma3(vab2, mbar, scale(pb, lbar));
  va = {R::fma(j, ibar.x, inner.x), R::fma(j, ibar.y, inner.y), R::fma(j, ibar.z, inner.z)};
  vb = sub(neg(va), pbar);
}

// One thread per (view, point): grad_points and the nine face terms (untouched vertices left unset),
// and the point counted in its (view, face) row.  A face index outside [0, F) contributes nothing.
template <typename T>
__global__ void __launch_bounds__(kThreads) pmd_point_grad_kernel(int N, int F, int64_t np, const T* __restrict__ grad_dist,
                                                                  const T* __restrict__ points, const T* __restrict__ fv,
                                                                  const int64_t* __restrict__ face_idx,
                                                                  const int32_t* __restrict__ dist_type,
                                                                  T* __restrict__ grad_points, T* __restrict__ terms,
                                                                  int* __restrict__ count) {
  using R = Rn<T>;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= np) return;
  const int64_t b = i / N, f = face_idx[i];
  if (f < 0 || f >= F) return;
  const int t = dist_type[i];
  const T* v = fv + (b * F + f) * 9;
  const V3<T> p = ld3(points + i * 3), v1 = ld3(v), v2 = ld3(v + 3), v3 = ld3(v + 6);
  const T g = grad_dist[i];
  const T go = R::add(g, g);   // 2. * grad_dist
  V3<T> gp, a1 = {}, a2 = {}, a3 = {};
  if (t == 0) {   // :342-373
    const V3<T> pv = sub(p, v1), e21 = sub(v1, v2), e31 = sub(v1, v3);
    const V3<T> normal = cross(e21, e31);
    const T len = R::sqrt(dot(normal, normal));
    const V3<T> un = {R::div(normal.x, len), R::div(normal.y, len), R::div(normal.z, len)};
    const T d = dot(pv, un);
    const V3<T> gdv = scale(un, R::mul(go, d));
    const T gd = dot(un, gdv);
    gp = scale(un, gd);
    const V3<T> gun = fma3(gdv, d, scale(pv, gd));
    const T q = R::div(dot(normal, gun), R::mul(len, len));
    const T gd2n = R::div(q, R::mul(len, T(-2)));
    const V3<T> gn = fma3(normal, R::add(gd2n, gd2n), V3<T>{R::div(gun.x, len), R::div(gun.y, len), R::div(gun.z, len)});
    const V3<T> ge31 = cross(gn, e21), ge21 = cross(e31, gn);
    a1 = sub(add(ge31, ge21), gp);
    a2 = neg(ge21);
    a3 = neg(ge31);
  } else if (t == 1) {
    gp = scale(sub(p, v1), go); a1 = neg(gp);
  } else if (t == 2) {
    gp = scale(sub(p, v2), go); a2 = neg(gp);
  } else if (t == 3) {
    gp = scale(sub(p, v3), go); a3 = neg(gp);
  } else if (t == 4) {
    edge_backward(sub(v2, v1), sub(p, v1), go, gp, a2, a1);
  } else if (t == 5) {
    edge_backward(sub(v3, v2), sub(p, v2), go, gp, a3, a2);
  } else {
    edge_backward(sub(v1, v3), sub(p, v3), go, gp, a1, a3);
  }
  if (grad_points) st3(grad_points + i * 3, gp);
  if (terms) {
    T* o = terms + i * 9;
    st3(o, a1); st3(o + 3, a2); st3(o + 6, a3);
    atomicAdd(count + b * F + f, 1);
  }
}

// Each point takes a slot of its (view, face) row, in whatever order the atomics give; the row sort
// puts the point ids in ascending order.
__global__ void __launch_bounds__(kThreads) pmd_fill_kernel(int N, int F, int64_t np, const int64_t* __restrict__ face_idx,
                                                            const int* __restrict__ off, int* __restrict__ count,
                                                            int* __restrict__ ids) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= np) return;
  const int64_t b = i / N, f = face_idx[i];
  if (f < 0 || f >= F) return;
  const int64_t row = b * F + f;
  ids[off[row] + atomicSub(count + row, 1) - 1] = (int)(i - b * N);
}

__global__ void __launch_bounds__(kThreads) pmd_sort_rows_kernel(int64_t rows, const int* __restrict__ off, int* __restrict__ ids,
                                                                 int* __restrict__ long_rows, int* __restrict__ long_count) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int b = off[r], n = off[r + 1] - b;
  if (n > kShortRow) {
    long_rows[atomicAdd(long_count, 1)] = (int)r;
    return;
  }
  insertion_sort(ids + b, n);
}

__global__ void __launch_bounds__(kSortThreads) pmd_sort_long_kernel(const int* __restrict__ off, int* __restrict__ ids,
                                                                     const int* __restrict__ long_rows,
                                                                     const int* __restrict__ long_count) {
  const int rows = *long_count;
  for (int k = blockIdx.x; k < rows; k += gridDim.x) {
    const int r = long_rows[k];
    block_bitonic_sort(ids + off[r], off[r + 1] - off[r]);
  }
}

// One thread per (view, face): its points' terms, in ascending point order, added onto the existing
// grad_face_vertices, each vertex only by the points whose type touches it.
template <typename T>
__global__ void __launch_bounds__(kThreads) pmd_face_grad_kernel(int N, int F, int64_t rows, const int* __restrict__ off,
                                                                 const int* __restrict__ ids,
                                                                 const int32_t* __restrict__ dist_type,
                                                                 const T* __restrict__ terms, T* __restrict__ gfv) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int b0 = off[r], b1 = off[r + 1];
  if (b0 == b1) return;
  const int64_t base = (r / F) * N;
  T acc[9];
  T* o = gfv + r * 9;
#pragma unroll
  for (int k = 0; k < 9; ++k) acc[k] = o[k];
  for (int s = b0; s < b1; ++s) {
    const int64_t i = base + ids[s];
    const int m = touched(dist_type[i]);
    const T* t = terms + i * 9;
#pragma unroll
    for (int k = 0; k < 9; ++k)
      if (m >> (k / 3) & 1) acc[k] = Rn<T>::acc(acc[k], t[k]);
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) o[k] = acc[k];
}

// ---------------------------------------------------------------------------------------------
// Host.

unsigned blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

size_t tsize_of(int dtype) {
  return dtype == DIBR_B200_DTYPE_F32 ? sizeof(float) : dtype == DIBR_B200_DTYPE_F64 ? sizeof(double) : 0;
}

// 0 or the error: the face index must fit the key's low 32 bits and every (view, point) and
// (view, face) index an int.
int check_dims(int B, int N, int F, int dtype) {
  if (B < 0 || N < 0 || F < 0 || tsize_of(dtype) == 0) return DIBR_B200_EINVAL;
  if ((int64_t)B * N >= 0x7fffffffLL || (int64_t)B * F >= 0x7fffffffLL) return DIBR_B200_ESIZE;
  return 0;
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev < 0 || dev >= 64) dev = 0;
  if (!cached[dev]) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cached[dev] = n > 0 ? n : 132;
  }
  return cached[dev];
}

template <typename T>
int forward(int B, int N, int F, const T* points, const T* fv, T* dist, int64_t* face_idx, int32_t* dist_type,
            char* o, const dibr_layout::PointMeshForwardLayout& L, cudaStream_t st) {
  const int64_t nf = (int64_t)B * F, np = (int64_t)B * N;
  T* rec = piece<T>(o, L.records);
  unsigned long long* keys = piece<unsigned long long>(o, L.keys);
  cudaError_t e = cudaMemsetAsync(keys, 0xFF, sizeof(unsigned long long) * (size_t)np, st);
  if (e != cudaSuccess) return (int)e;
  pmd_faces_kernel<T><<<blocks(nf, kThreads), kThreads, 0, st>>>(nf, fv, rec);
  // Face chunks: enough CTAs to fill the GPU when N is small, never a chunk under one tile.
  const int PB = (int)((N + kSearchPoints - 1) / kSearchPoints);
  const int64_t base = (int64_t)B * PB;
  const int64_t want = ((int64_t)kCtasPerSm * sm_count() + base - 1) / base;
  const int64_t most = (F + kTileFaces - 1) / kTileFaces;
  const int64_t C0 = want < 1 ? 1 : want > most ? most : want;
  const int chunk = (int)((F + C0 - 1) / C0);
  const int C = (F + chunk - 1) / chunk;
  pmd_search_kernel<T><<<(unsigned)(base * C), kSearchThreads, 0, st>>>(N, F, PB, C, chunk, points, rec, keys);
  pmd_finalize_kernel<T><<<blocks(np, kThreads), kThreads, 0, st>>>(N, F, points, rec, keys, dist, face_idx,
                                                                     dist_type, np);
  return (int)cudaGetLastError();
}

template <typename T>
int backward(int B, int N, int F, const T* grad_dist, const T* points, const T* fv, const int64_t* face_idx,
             const int32_t* dist_type, T* grad_points, T* gfv, char* o, const dibr_layout::PointMeshBackwardLayout& L,
             cudaStream_t st) {
  const int64_t np = (int64_t)B * N, rows = (int64_t)B * F;
  T* terms = gfv ? piece<T>(o, L.terms) : nullptr;
  int* count = piece<int>(o, L.count);
  int* off = piece<int>(o, L.off);
  int* ids = piece<int>(o, L.ids);
  int* long_rows = piece<int>(o, L.long_rows);
  int* long_count = piece<int>(o, L.long_count);
  if (gfv) {
    cudaError_t e = cudaMemsetAsync(count, 0, sizeof(int) * (size_t)(rows > 0 ? rows : 1), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(long_count, 0, sizeof(int), st);
    if (e != cudaSuccess) return (int)e;
  }
  pmd_point_grad_kernel<T><<<blocks(np, kThreads), kThreads, 0, st>>>(N, F, np, grad_dist, points, fv, face_idx, dist_type,
                                                                       grad_points, terms, count);
  if (!gfv || rows == 0) return (int)cudaGetLastError();
  if (int e = exclusive_scan(count, (int)rows, piece<int>(o, L.sums), off, st)) return e;
  pmd_fill_kernel<<<blocks(np, kThreads), kThreads, 0, st>>>(N, F, np, face_idx, off, count, ids);
  pmd_sort_rows_kernel<<<blocks(rows, kThreads), kThreads, 0, st>>>(rows, off, ids, long_rows, long_count);
  pmd_sort_long_kernel<<<kLongCtas, kSortThreads, 0, st>>>(off, ids, long_rows, long_count);
  pmd_face_grad_kernel<T><<<blocks(rows, kThreads), kThreads, 0, st>>>(N, F, rows, off, ids, dist_type, terms, gfv);
  return (int)cudaGetLastError();
}

}  // namespace

extern "C" {

int dibr_b200_point_mesh_distance_workspace_bytes(int batch, int num_points, int num_faces, int dtype,
                                                  size_t* forward_bytes, size_t* backward_bytes) {
  if (int r = check_dims(batch, num_points, num_faces, dtype)) return r;
  const size_t ts = tsize_of(dtype);
  if (forward_bytes) *forward_bytes = dibr_layout::point_mesh_forward_layout(batch, num_points, num_faces, ts).bytes;
  if (backward_bytes) *backward_bytes = dibr_layout::point_mesh_backward_layout(batch, num_points, num_faces, ts).bytes;
  return 0;
}

int dibr_b200_point_mesh_distance_forward(int batch, int num_points, int num_faces, int dtype, const void* points,
                                          const void* face_vertices, void* dist, int64_t* face_idx, int32_t* dist_type,
                                          void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream) {
  if (int r = check_dims(batch, num_points, num_faces, dtype)) return r;
  const int64_t np = (int64_t)batch * num_points;
  if (!workspace || (np > 0 && (!points || !dist || !face_idx || !dist_type)) ||
      ((int64_t)batch * num_faces > 0 && !face_vertices))
    return DIBR_B200_EINVAL;
  const dibr_layout::PointMeshForwardLayout L =
      dibr_layout::point_mesh_forward_layout(batch, num_points, num_faces, tsize_of(dtype));
  char* o = carve(workspace, workspace_bytes, L.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  if (np == 0 || num_faces == 0) return 0;   // no face: the outputs are left as they are
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == DIBR_B200_DTYPE_F32)
    return forward<float>(batch, num_points, num_faces, (const float*)points, (const float*)face_vertices,
                          (float*)dist, face_idx, dist_type, o, L, st);
  return forward<double>(batch, num_points, num_faces, (const double*)points, (const double*)face_vertices,
                         (double*)dist, face_idx, dist_type, o, L, st);
}

int dibr_b200_point_mesh_distance_backward(int batch, int num_points, int num_faces, int dtype, const void* grad_dist,
                                           const void* points, const void* face_vertices, const int64_t* face_idx,
                                           const int32_t* dist_type, void* grad_points, void* grad_face_vertices,
                                           void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream) {
  if (int r = check_dims(batch, num_points, num_faces, dtype)) return r;
  const int64_t np = (int64_t)batch * num_points;
  if (!workspace || (np > 0 && (!grad_dist || !points || !face_idx || !dist_type)) ||
      ((int64_t)batch * num_faces > 0 && !face_vertices))
    return DIBR_B200_EINVAL;
  const dibr_layout::PointMeshBackwardLayout L =
      dibr_layout::point_mesh_backward_layout(batch, num_points, num_faces, tsize_of(dtype));
  char* o = carve(workspace, workspace_bytes, L.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  if (np == 0 || num_faces == 0 || (!grad_points && !grad_face_vertices)) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == DIBR_B200_DTYPE_F32)
    return backward<float>(batch, num_points, num_faces, (const float*)grad_dist, (const float*)points,
                           (const float*)face_vertices, face_idx, dist_type, (float*)grad_points,
                           (float*)grad_face_vertices, o, L, st);
  return backward<double>(batch, num_points, num_faces, (const double*)grad_dist, (const double*)points,
                          (const double*)face_vertices, face_idx, dist_type, (double*)grad_points,
                          (double*)grad_face_vertices, o, L, st);
}

}  // extern "C"
