// voxelize.cu — kaolin.ops.conversions.trianglemeshes_to_voxelgrids and pointclouds_to_voxelgrids (the
// reference's kaolin/ops/conversions/trianglemesh.py:29-110 and pointcloud.py:22-141) for every view
// in one launch per kernel, behind the C ABI of include/dibr_b200.h.
//
// Points arrive normalised, (B, P, 3) float32 or float64 (T).  A point marks voxel
// (rint(x (res-1)), rint(y (res-1)), rint(z (res-1))) when all three lie in [0, res-1], tested in T
// before any conversion, so NaN and huge values are dropped.  The marks go to a bit grid of B res^3
// bits, bit ((b res + ix) res + iy) res + iz: the flat index of the dense output, 64-bit throughout.
//
// Meshes add the midpoints of the reference's subdivision (kaolin/ops/mesh/trianglemesh.py:340-458),
// with its rounding: a triangle (v1, v2, v3) is split when max(|v1-v2|^2, |v2-v3|^2, |v3-v1|^2) > thr,
// each squared length (dx dx + dy dy) + dz dz with every product and sum rounded on its own, thr
// = ((res-1)/res^2)^2 rounded to T.  A split marks m4 = (v1+v3)/2, m5 = (v1+v2)/2, m6 = (v2+v3)/2
// and recurses on (v1,m4,m5), (v2,m5,m6), (m4,m5,m6), (v3,m4,m6).  The point set does not depend on
// the order triangles are visited in, so each face is walked depth first on its own.  Every operation
// on this path is an _rn intrinsic: nothing is contracted or reassociated.
//
// Two rules keep the work bounded, and neither changes the point set:
//   - a triangle with a non-finite coordinate is not split (NaN: as the reference, whose max
//     propagates it; infinity: the reference never terminates there);
//   - range prune: a triangle whose three vertices all quantise below 0, or all above res-1, on one
//     axis is skipped.  fl((a+b)/2) lies in [min(a,b), max(a,b)] for finite a, b (an overflowing sum
//     is infinite, and such a triangle is not split), and quantisation is monotonic, so every
//     descendant lies in its ancestor's box and none of them could mark a voxel.
//
// Passes (all views at once): mark the points -> count (one thread per (view, face): index check,
// depth estimate d_f, 4^s_f work items, s_f = clamp(d_f - kItemLeafDepth, 0, S)) -> exclusive scan
// -> subdivide (one thread per item: descend s_f levels by the item's base-4 digits, then walk the
// rest depth first with an explicit stack of parents) -> dense expansion, or popcount per 32-word
// chunk, scan and emit of the sparse rows in grid order.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dibr_b200.h"
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

constexpr int kThreads = 256;
constexpr int kCtasPerSm = 8;
constexpr int kItemLeafDepth = 3;   // an item walks at least 4^3 leaves before faces are cut into items
constexpr int kMaxItemLevels = 9;   // S: a face becomes at most 4^9 items
constexpr int kMaxDepth = DIBR_B200_VOXELIZE_MAX_DEPTH;
constexpr int kStack = kMaxDepth + 2;   // parents on the walk's path; the estimate may be one level short

template <typename T> struct Fp;
template <> struct Fp<float> {
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float rnd(float a) { return rintf(a); }
};
template <> struct Fp<double> {
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
  static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
  static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
  static __device__ __forceinline__ double rnd(double a) { return rint(a); }
};

template <typename T>
struct Vox {
  int B, res;
  int64_t P, F, BF;      // points per view, faces, B F
  T rm1, thr;            // res - 1 and the split threshold, in T
  double thr_d;          // the same threshold, for the depth estimate
  int S;                 // most item levels a face is cut into
  const T* points;       // (B, P, 3)
  const int64_t* faces;  // (F, 3)
  uint32_t* bits;
  int* counts;           // (B F) work items per face
  const int* scan;       // (B F + 1)
  unsigned long long* info;   // {flags, first bad-index face, first too-deep face, nnz}
};

// The voxel of p along one axis, as a T: in range when 0 <= q <= res - 1 (false for NaN).
template <typename T>
__device__ __forceinline__ T quant(T p, T rm1) { return Fp<T>::rnd(Fp<T>::mul(p, rm1)); }

template <typename T>
__device__ __forceinline__ void mark(const Vox<T>& s, int b, T x, T y, T z) {
  const T qx = quant(x, s.rm1), qy = quant(y, s.rm1), qz = quant(z, s.rm1);
  if (!(qx >= T(0) && qx <= s.rm1 && qy >= T(0) && qy <= s.rm1 && qz >= T(0) && qz <= s.rm1)) return;
  const int64_t r = s.res;
  const int64_t id = (((int64_t)b * r + (int64_t)qx) * r + (int64_t)qy) * r + (int64_t)qz;
  uint32_t* w = s.bits + (id >> 5);
  const uint32_t m = 1u << (id & 31);
  if (!(*(volatile uint32_t*)w & m)) atomicOr(w, m);
}

template <typename T>
__device__ __forceinline__ T sq_edge(const T* a, const T* b) {
  using F = Fp<T>;
  const T dx = F::sub(a[0], b[0]), dy = F::sub(a[1], b[1]), dz = F::sub(a[2], b[2]);
  return F::add(F::add(F::mul(dx, dx), F::mul(dy, dy)), F::mul(dz, dz));
}

// Whether triangle t (v1, v2, v3 at t[0..8]) is split: finite, not range-pruned, longest squared edge
// above thr.  *m gets the longest squared edge when it is split.
template <typename T>
__device__ __forceinline__ bool splits(const Vox<T>& s, const T* t, T* m) {
#pragma unroll
  for (int k = 0; k < 9; ++k)
    if (!isfinite(t[k])) return false;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const T q0 = quant(t[a], s.rm1), q1 = quant(t[3 + a], s.rm1), q2 = quant(t[6 + a], s.rm1);
    if ((q0 < T(0) && q1 < T(0) && q2 < T(0)) || (q0 > s.rm1 && q1 > s.rm1 && q2 > s.rm1)) return false;
  }
  const T e12 = sq_edge(t, t + 3), e23 = sq_edge(t + 3, t + 6), e31 = sq_edge(t + 6, t);
  const T e = e12 > e23 ? e12 : e23, mx = e > e31 ? e : e31;
  *m = mx;
  return mx > s.thr;
}

template <typename T>
__device__ __forceinline__ void midpoints(const T* t, T* m) {
  using F = Fp<T>;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    m[a] = F::mul(F::add(t[a], t[6 + a]), T(0.5));          // m4 = (v1 + v3) / 2
    m[3 + a] = F::mul(F::add(t[a], t[3 + a]), T(0.5));      // m5 = (v1 + v2) / 2
    m[6 + a] = F::mul(F::add(t[3 + a], t[6 + a]), T(0.5));  // m6 = (v2 + v3) / 2
  }
}

template <typename T>
__device__ __forceinline__ void mark_midpoints(const Vox<T>& s, int b, const T* m) {
  mark(s, b, m[0], m[1], m[2]);
  mark(s, b, m[3], m[4], m[5]);
  mark(s, b, m[6], m[7], m[8]);
}

// Child k of t, from t's midpoints m: (v1,m4,m5), (v2,m5,m6), (m4,m5,m6), (v3,m4,m6).
template <typename T>
__device__ __forceinline__ void child(const T* t, const T* m, int k, T* c) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const T v1 = t[a], v2 = t[3 + a], v3 = t[6 + a], m4 = m[a], m5 = m[3 + a], m6 = m[6 + a];
    c[a] = k == 0 ? v1 : k == 1 ? v2 : k == 2 ? m4 : v3;
    c[3 + a] = k == 0 ? m4 : k == 1 ? m5 : k == 2 ? m5 : m4;
    c[6 + a] = k == 0 ? m5 : k == 1 ? m6 : k == 2 ? m6 : m6;
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) vox_mark_points_kernel(Vox<T> s) {
  const int64_t n = (int64_t)s.B * s.P;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const T* p = s.points + 3 * i;
    mark(s, (int)(i / s.P), p[0], p[1], p[2]);
  }
}

// The face's three vertices, or false when an index lies outside [0, P).
template <typename T>
__device__ __forceinline__ bool load_face(const Vox<T>& s, int64_t q, T* t) {
  const int64_t b = q / s.F, f = q - b * s.F;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int64_t v = __ldg(s.faces + 3 * f + k);
    if (v < 0 || v >= s.P) return false;
    const T* p = s.points + 3 * (b * s.P + v);
    t[3 * k] = p[0];
    t[3 * k + 1] = p[1];
    t[3 * k + 2] = p[2];
  }
  return true;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) vox_count_kernel(Vox<T> s) {
  for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < s.BF; q += (int64_t)gridDim.x * blockDim.x) {
    T t[9], m;
    int items = 0;
    if (!load_face(s, q, t)) {
      atomicOr(s.info, (unsigned long long)DIBR_B200_VOXELIZE_BAD_INDEX);
      atomicMin(s.info + 1, (unsigned long long)q);
    } else if (splits(s, t, &m)) {
      // levels until the longest squared edge, quartered per level, is at most thr
      double e = (double)m;
      int d = 0;
      while (e > s.thr_d && d <= kMaxDepth) { e *= 0.25; ++d; }
      if (d > kMaxDepth) {
        atomicOr(s.info, (unsigned long long)DIBR_B200_VOXELIZE_TOO_DEEP);
        atomicMin(s.info + 2, (unsigned long long)q);
      } else {
        const int lv = min(max(d - kItemLeafDepth, 0), s.S);
        items = 1 << (2 * lv);
      }
    }
    s.counts[q] = items;
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) vox_subdivide_kernel(Vox<T> s) {
  const int total = __ldg(s.scan + s.BF);
  for (int item = blockIdx.x * blockDim.x + threadIdx.x; item < total; item += gridDim.x * blockDim.x) {
    // the face: the last q with scan[q] <= item
    int64_t lo = 0, hi = s.BF;
    while (hi - lo > 1) {
      const int64_t mid = (lo + hi) >> 1;
      if (__ldg(s.scan + mid) <= item) lo = mid; else hi = mid;
    }
    const int64_t q = lo;
    const int j = item - __ldg(s.scan + q), n = __ldg(s.scan + q + 1) - __ldg(s.scan + q);
    const int lv = (31 - __clz(n)) >> 1;
    const int b = (int)(q / s.F);
    T t[9], m[9], c[9], e;
    load_face(s, q, t);   // faces with items have valid indices
    // descend lv levels by j's base-4 digits; the item whose digits from this level down are all zero
    // marks the node's midpoints
    bool alive = true;
    for (int l = 0; l < lv; ++l) {
      if (!splits(s, t, &e)) { alive = false; break; }
      midpoints(t, m);
      if ((j & ((1 << (2 * (lv - l))) - 1)) == 0) mark_midpoints(s, b, m);
      child(t, m, (j >> (2 * (lv - 1 - l))) & 3, c);
#pragma unroll
      for (int k = 0; k < 9; ++k) t[k] = c[k];
    }
    if (!alive) continue;
    // depth first below: stack[d] is the parent at depth d of the walk, 2 bits per depth its child
    T stack[kStack][9];
    uint64_t path = 0;
    int top = 0;
    while (true) {
      if (splits(s, t, &e)) {
        midpoints(t, m);
        mark_midpoints(s, b, m);
        if (top == kStack) {
          atomicOr(s.info, (unsigned long long)DIBR_B200_VOXELIZE_TOO_DEEP);
          atomicMin(s.info + 2, (unsigned long long)q);
        } else {
#pragma unroll
          for (int k = 0; k < 9; ++k) stack[top][k] = t[k];
          path &= ~(3ull << (2 * top));
          ++top;
          child(stack[top - 1], m, 0, c);
#pragma unroll
          for (int k = 0; k < 9; ++k) t[k] = c[k];
          continue;
        }
      }
      while (top > 0 && ((path >> (2 * (top - 1))) & 3) == 3) --top;
      if (top == 0) break;
      path += 1ull << (2 * (top - 1));
      midpoints(stack[top - 1], m);
      child(stack[top - 1], m, (int)((path >> (2 * (top - 1))) & 3), c);
#pragma unroll
      for (int k = 0; k < 9; ++k) t[k] = c[k];
    }
  }
}

// Dense: element i of the (B, res, res, res) output is bit i; one thread per 16 bytes of output.
template <typename T>
__global__ void __launch_bounds__(kThreads) vox_dense_kernel(const uint32_t* __restrict__ bits, int64_t n, T* out) {
  constexpr int kVec = 16 / sizeof(T);
  const int64_t nvec = (n + kVec - 1) / kVec;
  for (int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; v < nvec; v += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e = v * kVec;
    const uint32_t w = __ldg(bits + (e >> 5)) >> (e & 31);
    if (e + kVec <= n) {
      if constexpr (kVec == 4) {
        reinterpret_cast<float4*>(out)[v] = make_float4(w & 1, (w >> 1) & 1, (w >> 2) & 1, (w >> 3) & 1);
      } else {
        reinterpret_cast<double2*>(out)[v] = make_double2(w & 1, (w >> 1) & 1);
      }
    } else {
      for (int k = 0; e + k < n; ++k) out[e + k] = (T)((w >> k) & 1);
    }
  }
}

// Sparse, pass 1: the set bits of each chunk of 32 words (one warp) and their total.
__global__ void __launch_bounds__(kThreads) vox_chunk_count_kernel(const uint32_t* __restrict__ bits, int64_t nwords,
                                                                    int64_t nchunks, int* chunk_counts,
                                                                    unsigned long long* nnz) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t c = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; c < nchunks; c += warps) {
    const int64_t w = 32 * c + lane;
    int k = w < nwords ? __popc(__ldg(bits + w)) : 0;
#pragma unroll
    for (int o = 16; o; o >>= 1) k += __shfl_xor_sync(0xffffffffu, k, o);
    if (lane == 0) {
      chunk_counts[c] = k;
      if (k) atomicAdd(nnz, (unsigned long long)k);
    }
  }
}

// Sparse, pass 2: each set bit's (b, x, y, z) at its rank in grid order, rows of the (4, nnz) output.
__global__ void __launch_bounds__(kThreads) vox_emit_kernel(const uint32_t* __restrict__ bits, int64_t nwords,
                                                             int64_t nchunks, int res, const int* chunk_scan,
                                                             int64_t nnz, int64_t* out) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t c = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; c < nchunks; c += warps) {
    const int64_t w = 32 * c + lane;
    uint32_t word = w < nwords ? __ldg(bits + w) : 0u;
    const int k = __popc(word);
    int incl = k;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    int64_t at = (int64_t)__ldg(chunk_scan + c) + incl - k;
    while (word) {
      const int bit = __ffs(word) - 1;
      word &= word - 1;
      int64_t id = 32 * w + bit;
      const int64_t z = id % res;
      id /= res;
      const int64_t y = id % res;
      id /= res;
      const int64_t x = id % res;
      out[at] = id / res;
      out[nnz + at] = x;
      out[2 * nnz + at] = y;
      out[3 * nnz + at] = z;
      ++at;
    }
  }
}

unsigned grid_stride_ctas(int64_t n) {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  const int64_t need = (n + kThreads - 1) / kThreads, cap = (int64_t)sms * kCtasPerSm;
  return (unsigned)(need < 1 ? 1 : need < cap ? need : cap);
}

struct Shape {
  int64_t BF, bits, nwords, nchunks;
};

// Sizes and their limits: B F, the items of B F faces and the chunk counts are indexed by int.
int vox_shape(int batch, int64_t num_faces, int res, Shape* sh) {
  if (batch < 0 || num_faces < 0 || res < 1) return DIBR_B200_EINVAL;
  const int64_t r3 = (int64_t)res * res * res;
  if (res > (1 << 20) || (batch > 0 && r3 > (INT64_MAX >> 8) / batch)) return DIBR_B200_ESIZE;
  sh->BF = (int64_t)batch * num_faces;
  sh->bits = (int64_t)batch * r3;
  sh->nwords = (sh->bits + 31) / 32;
  sh->nchunks = (sh->nwords + 31) / 32;
  if (sh->BF >= INT32_MAX || sh->nchunks >= INT32_MAX) return DIBR_B200_ESIZE;
  return 0;
}

dibr_layout::VoxelizeLayout vox_layout(const Shape& sh) {
  return dibr_layout::voxelize_layout(sh.nwords, sh.BF, sh.nchunks);
}

template <typename T>
int vox_mark(int batch, int64_t num_points, int64_t num_faces, int res, const void* points, const int64_t* faces,
             int sparse, int64_t* info, const Shape& sh, char* o, cudaStream_t st) {
  const dibr_layout::VoxelizeLayout L = vox_layout(sh);
  Vox<T> s{};
  s.B = batch; s.res = res; s.P = num_points; s.F = num_faces; s.BF = sh.BF;
  s.rm1 = (T)(res - 1);
  const double thr = ((double)(res - 1) / ((double)res * res)) * ((double)(res - 1) / ((double)res * res));
  s.thr = (T)thr;
  s.thr_d = (double)s.thr;
  int S = 0;   // B F 4^S items stay below 2^31
  while (S < kMaxItemLevels && (sh.BF << (2 * (S + 1))) < INT32_MAX) ++S;
  s.S = S;
  s.points = (const T*)points;
  s.faces = faces;
  s.bits = dibr_layout::piece<uint32_t>(o, L.bits);
  s.counts = dibr_layout::piece<int>(o, L.counts);
  s.scan = dibr_layout::piece<int>(o, L.scan);
  s.info = (unsigned long long*)info;
  if (cudaMemsetAsync(info, 0, sizeof(int64_t), st) || cudaMemsetAsync(info + 1, 0xff, 2 * sizeof(int64_t), st) ||
      cudaMemsetAsync(info + 3, 0, sizeof(int64_t), st) || cudaMemsetAsync(s.bits, 0, 4 * sh.nwords, st))
    return (int)cudaGetLastError();
  if ((int64_t)batch * num_points > 0) {
    Span sp("vox_mark_points_kernel", st);
    vox_mark_points_kernel<T><<<grid_stride_ctas((int64_t)batch * num_points), kThreads, 0, st>>>(s);
  }
  if (sh.BF > 0) {
    { Span sp("vox_count_kernel", st); vox_count_kernel<T><<<grid_stride_ctas(sh.BF), kThreads, 0, st>>>(s); }
    if (int e = dibr_b200_detail::exclusive_scan(s.counts, (int)sh.BF, dibr_layout::piece<int>(o, L.sums),
                                                 dibr_layout::piece<int>(o, L.scan), st))
      return e;
    // enough CTAs to fill the GPU; each thread strides over the items
    Span sp("vox_subdivide_kernel", st);
    vox_subdivide_kernel<T><<<grid_stride_ctas(INT32_MAX), kThreads, 0, st>>>(s);
  }
  if (sparse) {
    int* cc = dibr_layout::piece<int>(o, L.chunk_counts);
    {
      Span sp("vox_chunk_count_kernel", st);
      vox_chunk_count_kernel<<<grid_stride_ctas(32 * sh.nchunks), kThreads, 0, st>>>(
          s.bits, sh.nwords, sh.nchunks, cc, (unsigned long long*)info + 3);
    }
    if (int e = dibr_b200_detail::exclusive_scan(cc, (int)sh.nchunks, dibr_layout::piece<int>(o, L.sums),
                                                 dibr_layout::piece<int>(o, L.chunk_scan), st))
      return e;
  }
  return (int)cudaGetLastError();
}

}  // namespace

int dibr_b200_voxelize_workspace_bytes(int batch, int64_t num_faces, int resolution, size_t* workspace_bytes) {
  if (!workspace_bytes) return DIBR_B200_EINVAL;
  Shape sh;
  if (const int e = vox_shape(batch, num_faces, resolution, &sh)) return e;
  *workspace_bytes = vox_layout(sh).bytes;
  return 0;
}

int dibr_b200_voxelize_mark(int batch, int64_t num_points, int64_t num_faces, int resolution, int dtype,
                            const void* points, const int64_t* faces, int sparse, int64_t* info, void* workspace,
                            size_t workspace_bytes, dibr_b200_stream_t stream) {
  Shape sh;
  if (const int e = vox_shape(batch, num_faces, resolution, &sh)) return e;
  if (num_points < 0 || (dtype != DIBR_B200_DTYPE_F32 && dtype != DIBR_B200_DTYPE_F64)) return DIBR_B200_EINVAL;
  if (!info || (batch > 0 && num_points > 0 && !points) || (num_faces > 0 && !faces)) return DIBR_B200_EINVAL;
  char* o = dibr_layout::carve(workspace, workspace_bytes, vox_layout(sh).bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  return dtype == DIBR_B200_DTYPE_F32
             ? vox_mark<float>(batch, num_points, num_faces, resolution, points, faces, sparse, info, sh, o, st)
             : vox_mark<double>(batch, num_points, num_faces, resolution, points, faces, sparse, info, sh, o, st);
}

int dibr_b200_voxelize_dense(int batch, int64_t num_faces, int resolution, int dtype, void* out, void* workspace,
                             size_t workspace_bytes, dibr_b200_stream_t stream) {
  Shape sh;
  if (const int e = vox_shape(batch, num_faces, resolution, &sh)) return e;
  if (dtype != DIBR_B200_DTYPE_F32 && dtype != DIBR_B200_DTYPE_F64) return DIBR_B200_EINVAL;
  if (sh.bits == 0) return 0;
  if (!out || ((uintptr_t)out & 15)) return DIBR_B200_EINVAL;
  const dibr_layout::VoxelizeLayout L = vox_layout(sh);
  char* o = dibr_layout::carve(workspace, workspace_bytes, L.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const uint32_t* bits = dibr_layout::piece<uint32_t>(o, L.bits);
  const int64_t nvec = dtype == DIBR_B200_DTYPE_F32 ? (sh.bits + 3) / 4 : (sh.bits + 1) / 2;
  Span sp("vox_dense_kernel", st);
  if (dtype == DIBR_B200_DTYPE_F32)
    vox_dense_kernel<float><<<grid_stride_ctas(nvec), kThreads, 0, st>>>(bits, sh.bits, (float*)out);
  else
    vox_dense_kernel<double><<<grid_stride_ctas(nvec), kThreads, 0, st>>>(bits, sh.bits, (double*)out);
  return (int)cudaGetLastError();
}

int dibr_b200_voxelize_sparse(int batch, int64_t num_faces, int resolution, int64_t nnz, int64_t* out_indices,
                              void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream) {
  Shape sh;
  if (const int e = vox_shape(batch, num_faces, resolution, &sh)) return e;
  if (nnz < 0 || nnz > INT32_MAX) return DIBR_B200_ESIZE;
  if (nnz == 0) return 0;
  if (!out_indices) return DIBR_B200_EINVAL;
  const dibr_layout::VoxelizeLayout L = vox_layout(sh);
  char* o = dibr_layout::carve(workspace, workspace_bytes, L.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  Span sp("vox_emit_kernel", st);
  vox_emit_kernel<<<grid_stride_ctas(32 * sh.nchunks), kThreads, 0, st>>>(
      dibr_layout::piece<uint32_t>(o, L.bits), sh.nwords, sh.nchunks, resolution,
      dibr_layout::piece<int>(o, L.chunk_scan), nnz, out_indices);
  return (int)cudaGetLastError();
}
