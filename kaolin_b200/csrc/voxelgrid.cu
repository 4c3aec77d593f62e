// voxelgrid.cu — kaolin.ops.voxelgrid (the reference's kaolin/ops/voxelgrid.py): fill, extract_surface,
// extract_odms and project_odms for every view in one launch per kernel, behind the C ABI of
// include/dibr_b200.h.  Grids are (batch, X, Y, Z), read in place through element strides; a voxel is
// occupied when its value is nonzero (NaN is, -0.0 is not).
//
// fill: the empty voxels whose 6-connected empty component touches no border face become occupied
// (scipy.ndimage.binary_fill_holes with its default structure).  Union-find over the empty voxels of
// each view, in the style of Playne & Hawick (IEEE TPDS 2018):
//   - labels [batch][X Y Z] int32 in the workspace: -1 for an occupied voxel, else a node id.  Node
//     v + 1 is voxel v of the view; node 0 is OUTSIDE and has no slot.  A node's parent always has a
//     smaller id, so the forest has no cycle and a component's root is its smallest node;
//   - init: every empty voxel points at the first voxel of its run along z, which is the run's root,
//     so runs start merged;
//   - merge: each overlapping segment of two runs adjacent in x or y is merged once, at its first z,
//     with the lock-free atomicMin union; every run that touches a border face is merged with
//     OUTSIDE.  OUTSIDE, the smallest node, becomes the root of every component reaching the border;
//   - output: occupied || find(v) != 0, 16 voxels per thread and one 16-byte store.
// find halves paths as it walks.  Every pointer it writes is an ancestor, and a union that loses a
// race to it retries with the node's new parent, so the components and the output do not depend on
// the order the atomics run in.  The launches are three whatever the content.
//
// extract_surface: a 3x3x3 stencil over three x planes staged in shared memory.  Float grids sum the
// in-bounds values in T in the loop order of torch's CUDA avg_pool3d (x outer, z inner), divide by 27
// (wide) or by 3 (thin, one window per axis) with _rn, and compare with 1, so the predicate is
// bit-equal to the reference's; bool grids count the occupied neighbours.
//
// extract_odms: one pass over the grid.  A CTA takes an 8 x 8 tile of (x, y) rows and walks z in warp
// chunks: each row's first and last occupied z come from ballots, the first and last y of each (x, z)
// and the first and last x of each (y, z) are reduced in registers and shared memory, and each CTA adds
// them to the maps with one integer atomicMin per (map, column).
//
// project_odms: one thread per voxel, the six masks in the dtype torch's type promotion gives the
// reference.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dibr_b200.h"
#include "op_layouts.h"

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

unsigned grid_stride_ctas(int64_t n, int per_cta = kThreads) {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  const int64_t need = (n + per_cta - 1) / per_cta, cap = (int64_t)sms * kCtasPerSm;
  return (unsigned)(need < 1 ? 1 : need < cap ? need : cap);
}

// A strided (batch, X, Y, Z) grid of T.
template <typename T>
struct Grid {
  const T* p;
  int64_t sb, sx, sy, sz;
  __device__ __forceinline__ T at(int64_t b, int x, int y, int z) const {
    return p[b * sb + x * sx + y * sy + z * sz];
  }
};

template <typename T>
__device__ __forceinline__ bool occupied(T v) { return v != T(0); }

// ---------------------------------------------------------------------------------------------
// fill

// The root of node a (0 for OUTSIDE), halving the path on the way.
__device__ __forceinline__ int find_root(volatile int* L, int a) {
  while (a != 0) {
    const int p = L[a - 1];
    if (p == a) return a;
    if (p == 0) return 0;
    const int g = L[p - 1];
    if (g == p) return p;
    L[a - 1] = g;
    a = g;
  }
  return 0;
}

// Merges the components of nodes a and b: the larger root is linked under the smaller one.  If the
// larger root gained a parent meanwhile, atomicMin may have re-pointed it, so the union is retried
// with the parent it had.
__device__ __forceinline__ void unite(volatile int* L, int a, int b) {
  while (true) {
    a = find_root(L, a);
    b = find_root(L, b);
    if (a == b) return;
    if (a < b) { const int t = a; a = b; b = t; }
    const int old = atomicMin((int*)&L[a - 1], b);
    if (old == a) return;
    a = old;
  }
}

struct FillShape {
  int64_t B, rows;   // views, (view, x, y) rows
  int X, Y, Z, N;    // N = X Y Z voxels per view
};

// One warp per (view, x, y) row, 32 z at a time: each empty voxel gets its run's first voxel, found
// from the ballot of run starts and the run carried in from the previous chunk.
template <typename T>
__global__ void __launch_bounds__(kThreads) vg_fill_init_kernel(Grid<T> g, FillShape s, int* __restrict__ L) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; r < s.rows; r += warps) {
    const int64_t b = r / ((int64_t)s.X * s.Y);
    const int xy = (int)(r - b * s.X * s.Y), x = xy / s.Y, y = xy - x * s.Y;
    int* dst = L + r * s.Z;
    const int row = xy * s.Z;   // the view's voxel index of (x, y, 0)
    int carry_start = 0;
    bool carry_empty = false;
    for (int z0 = 0; z0 < s.Z; z0 += 32) {
      const int z = z0 + lane;
      const bool in = z < s.Z;
      const bool empty = in && !occupied(g.at(b, x, y, z));
      const unsigned em = __ballot_sync(0xffffffffu, empty);
      const unsigned starts = em & ~((em << 1) | (carry_empty ? 1u : 0u));
      const unsigned upto = starts & (0xffffffffu >> (31 - lane));
      const int start = upto ? z0 + 31 - __clz(upto) : carry_start;
      if (in) dst[z] = empty ? row + start + 1 : -1;
      carry_start = __shfl_sync(0xffffffffu, start, 31);
      carry_empty = (em >> 31) & 1u;
    }
  }
}

// One warp per row: merges each segment shared with the -x and -y rows at its first z, and every run
// on a border face with OUTSIDE.  Emptiness is read from the labels' sign, which no union changes.
__global__ void __launch_bounds__(kThreads) vg_fill_merge_kernel(FillShape s, int* L) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int YZ = s.Y * s.Z;
  for (int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; r < s.rows; r += warps) {
    const int64_t b = r / ((int64_t)s.X * s.Y);
    const int xy = (int)(r - b * s.X * s.Y), x = xy / s.Y, y = xy - x * s.Y;
    volatile int* Lb = L + b * s.N;
    const bool side = x == 0 || x == s.X - 1 || y == 0 || y == s.Y - 1;
    for (int z = lane; z < s.Z; z += 32) {
      const int v = xy * s.Z + z;
      const int l = Lb[v];
      if (l < 0) continue;
      const bool run_start = z == 0 || Lb[v - 1] < 0;
      if (x > 0) {
        const int n = Lb[v - YZ];
        if (n >= 0 && (run_start || Lb[v - YZ - 1] < 0)) unite(Lb, l, n);
      }
      if (y > 0) {
        const int n = Lb[v - s.Z];
        if (n >= 0 && (run_start || Lb[v - s.Z - 1] < 0)) unite(Lb, l, n);
      }
      if (z == s.Z - 1 || (run_start && (side || z == 0))) unite(Lb, l, 0);
    }
  }
}

// 16 voxels per thread in flat (view, voxel) order: occupied, or a root other than OUTSIDE.
__global__ void __launch_bounds__(kThreads) vg_fill_output_kernel(FillShape s, int* L, uint8_t* __restrict__ out) {
  const int64_t total = s.B * s.N, groups = (total + 15) / 16;
  for (int64_t gi = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; gi < groups;
       gi += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i0 = 16 * gi;
    int64_t base = i0 / s.N * s.N;
    uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const int64_t i = i0 + k;
      if (i < total) {
        while (i - base >= s.N) base += s.N;
        const int l = ((volatile int*)L)[i];
        const bool on = l < 0 || find_root(L + base, l) != 0;
        w[k >> 2] |= (uint32_t)on << (8 * (k & 3));
      }
    }
    if (i0 + 16 <= total) {
      *(uint4*)(out + i0) = make_uint4(w[0], w[1], w[2], w[3]);
    } else {
#pragma unroll
      for (int k = 0; k < 16; ++k)
        if (i0 + k < total) out[i0 + k] = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
    }
  }
}

// ---------------------------------------------------------------------------------------------
// extract_surface

constexpr int kSurfZ = 32, kSurfY = 8, kSurfX = 16;   // tile: z per warp, y rows per CTA, x planes walked

template <typename T> struct Acc;
template <> struct Acc<uint8_t> {   // bool: the count of occupied voxels
  using type = int;
  static __device__ __forceinline__ int add(int s, uint8_t v) { return s + (v != 0); }
  static __device__ __forceinline__ bool below(int s, int n) { return s < n; }
};
template <> struct Acc<float> {
  using type = float;
  static __device__ __forceinline__ float add(float s, float v) { return __fadd_rn(s, v); }
  static __device__ __forceinline__ bool below(float s, int n) { return __fdiv_rn(s, (float)n) < 1.f; }
};
template <> struct Acc<double> {
  using type = double;
  static __device__ __forceinline__ double add(double s, double v) { return __dadd_rn(s, v); }
  static __device__ __forceinline__ bool below(double s, int n) { return __ddiv_rn(s, (double)n) < 1.0; }
};

struct SurfShape {
  int64_t B, tiles;
  int X, Y, Z, tx, ty, tz;   // tiles per axis
};

// A CTA of 32 x 8 threads walks kSurfX x planes of one (view, y, z) tile, three planes (with a one-voxel
// zero halo, which adds nothing to a sum that starts at +0) in a shared ring.
template <typename T, bool kThin>
__global__ void __launch_bounds__(kSurfZ * kSurfY) vg_surface_kernel(Grid<T> g, SurfShape s,
                                                                     uint8_t* __restrict__ out) {
  using A = Acc<T>;
  using S = typename A::type;
  __shared__ T ring[3][kSurfY + 2][kSurfZ + 2];
  const int tz = threadIdx.x, ty = threadIdx.y, tid = ty * kSurfZ + tz;
  constexpr int kPlane = (kSurfY + 2) * (kSurfZ + 2);
  for (int64_t t = blockIdx.x; t < s.tiles; t += gridDim.x) {
    int64_t q = t;
    const int cz = (int)(q % s.tz); q /= s.tz;
    const int cy = (int)(q % s.ty); q /= s.ty;
    const int cx = (int)(q % s.tx);
    const int64_t b = q / s.tx;
    const int x0 = cx * kSurfX, y0 = cy * kSurfY, z0 = cz * kSurfZ;
    const int x1 = min(x0 + kSurfX, s.X);
    auto load = [&](int x) {
      T* dst = &ring[(x + 3) % 3][0][0];
      for (int k = tid; k < kPlane; k += kSurfZ * kSurfY) {
        const int yy = y0 - 1 + k / (kSurfZ + 2), zz = z0 - 1 + k % (kSurfZ + 2);
        const bool in = x >= 0 && x < s.X && yy >= 0 && yy < s.Y && zz >= 0 && zz < s.Z;
        dst[k] = in ? g.at(b, x, yy, zz) : T(0);
      }
    };
    load(x0 - 1);
    load(x0);
    const int y = y0 + ty, z = z0 + tz;
    for (int x = x0; x < x1; ++x) {
      load(x + 1);
      __syncthreads();
      const T c = ring[x % 3][ty + 1][tz + 1];
      bool keep;
      if (kThin) {
        S sx = S(0), sy = S(0), sz = S(0);
#pragma unroll
        for (int d = -1; d <= 1; ++d) {
          sx = A::add(sx, ring[(x + d + 3) % 3][ty + 1][tz + 1]);
          sy = A::add(sy, ring[x % 3][ty + 1 + d][tz + 1]);
          sz = A::add(sz, ring[x % 3][ty + 1][tz + 1 + d]);
        }
        keep = A::below(sx, 3) || A::below(sy, 3) || A::below(sz, 3);
      } else {
        S sum = S(0);
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx)
#pragma unroll
          for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
            for (int dz = -1; dz <= 1; ++dz) sum = A::add(sum, ring[(x + dx + 3) % 3][ty + 1 + dy][tz + 1 + dz]);
        keep = A::below(sum, 27);
      }
      if (y < s.Y && z < s.Z)
        out[((b * s.X + x) * s.Y + y) * (int64_t)s.Z + z] = (uint8_t)(keep && occupied(c));
      __syncthreads();
    }
  }
}

// ---------------------------------------------------------------------------------------------
// extract_odms: out (batch, 6, D, D) int64; map 2k+1 holds the first occupied voxel along its axis
// and map 2k the empty voxels after the last one, D where a ray meets none.

__global__ void vg_odms_init_kernel(int64_t n, int64_t D, long long* out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = D;
}

constexpr int kOdmTile = 8;   // (x, y) rows per CTA side; one warp per x

template <typename T>
__global__ void __launch_bounds__(32 * kOdmTile) vg_odms_kernel(Grid<T> g, int64_t B, int D, long long* out) {
  __shared__ int xlo[kOdmTile][32], xhi[kOdmTile][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int t1 = (D + kOdmTile - 1) / kOdmTile;
  const int64_t tiles = B * t1 * t1;
  const int64_t DD = (int64_t)D * D;
  for (int i = threadIdx.x; i < kOdmTile * 32; i += blockDim.x) {
    xlo[i / 32][i % 32] = INT32_MAX;
    xhi[i / 32][i % 32] = -1;
  }
  __syncthreads();
  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int64_t b = t / ((int64_t)t1 * t1);
    const int rem = (int)(t - b * t1 * t1);
    const int x = (rem / t1) * kOdmTile + w, y0 = (rem % t1) * kOdmTile;
    long long* ob = out + b * 6 * DD;
    int zlo[kOdmTile], zhi[kOdmTile];
#pragma unroll
    for (int k = 0; k < kOdmTile; ++k) { zlo[k] = INT32_MAX; zhi[k] = -1; }
    for (int z0 = 0; z0 < D; z0 += 32) {
      const int z = z0 + lane;
      int ylo = INT32_MAX, yhi = -1;
#pragma unroll
      for (int k = 0; k < kOdmTile; ++k) {
        const int y = y0 + k;
        const bool occ = x < D && y < D && z < D && occupied(g.at(b, x, y, z));
        const unsigned m = __ballot_sync(0xffffffffu, occ);
        if (m) {
          zlo[k] = min(zlo[k], z0 + __ffs(m) - 1);
          zhi[k] = max(zhi[k], z0 + 31 - __clz(m));
        }
        if (occ) {
          ylo = min(ylo, y);
          yhi = max(yhi, y);
          atomicMin_block(&xlo[k][lane], x);
          atomicMax_block(&xhi[k][lane], x);
        }
      }
      if (yhi >= 0) {
        const int64_t at = (int64_t)x * D + z;
        atomicMin(ob + 3 * DD + at, (long long)ylo);
        atomicMin(ob + 2 * DD + at, (long long)(D - 1 - yhi));
      }
      __syncthreads();
      {
        const int k = threadIdx.x >> 5;   // y0 + k, z0 + lane
        if (xhi[k][lane] >= 0) {
          const int64_t at = (int64_t)(y0 + k) * D + z0 + lane;
          atomicMin(ob + 5 * DD + at, (long long)xlo[k][lane]);
          atomicMin(ob + 4 * DD + at, (long long)(D - 1 - xhi[k][lane]));
          xlo[k][lane] = INT32_MAX;
          xhi[k][lane] = -1;
        }
      }
      __syncthreads();
    }
    if (lane < kOdmTile && x < D && y0 + lane < D) {
      int lo = zlo[0], hi = zhi[0];
#pragma unroll
      for (int k = 1; k < kOdmTile; ++k)
        if (lane == k) { lo = zlo[k]; hi = zhi[k]; }
      const int64_t at = (int64_t)x * D + y0 + lane;
      ob[DD + at] = hi >= 0 ? lo : D;
      ob[at] = hi >= 0 ? D - 1 - hi : D;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// project_odms

// dim - odm in the odms' dtype (integers wrap) and the comparisons with an int64 index under torch's
// promotion: integer odms compare as int64, float odms in their own type.
template <typename O> struct Odm;
template <> struct Odm<int64_t> {
  static __device__ __forceinline__ int64_t rsub(int64_t d, int64_t o) { return (int64_t)((uint64_t)d - (uint64_t)o); }
  static __device__ __forceinline__ bool ge(int i, int64_t o) { return (int64_t)i >= o; }
  static __device__ __forceinline__ bool lt(int i, int64_t o) { return (int64_t)i < o; }
};
template <> struct Odm<int32_t> {
  static __device__ __forceinline__ int32_t rsub(int64_t d, int32_t o) { return (int32_t)((uint32_t)d - (uint32_t)o); }
  static __device__ __forceinline__ bool ge(int i, int32_t o) { return (int64_t)i >= (int64_t)o; }
  static __device__ __forceinline__ bool lt(int i, int32_t o) { return (int64_t)i < (int64_t)o; }
};
template <> struct Odm<float> {
  static __device__ __forceinline__ float rsub(int64_t d, float o) { return __fsub_rn((float)d, o); }
  static __device__ __forceinline__ bool ge(int i, float o) { return (float)i >= o; }
  static __device__ __forceinline__ bool lt(int i, float o) { return (float)i < o; }
};
template <> struct Odm<double> {
  static __device__ __forceinline__ double rsub(int64_t d, double o) { return __dsub_rn((double)d, o); }
  static __device__ __forceinline__ bool ge(int i, double o) { return (double)i >= o; }
  static __device__ __forceinline__ bool lt(int i, double o) { return (double)i < o; }
};

// voxel * votes - count > 0 in the reference's result dtype.
enum GridKind { kAllOnes, kBool, kU8, kF32, kF64 };
template <int K> struct Vote;
template <> struct Vote<kAllOnes> {
  using T = uint8_t;
  static __device__ __forceinline__ bool keep(const Grid<T>&, int64_t, int, int, int, int64_t votes, int c) {
    return votes - c > 0;
  }
};
template <> struct Vote<kBool> {
  using T = uint8_t;
  static __device__ __forceinline__ bool keep(const Grid<T>& g, int64_t b, int x, int y, int z, int64_t votes, int c) {
    return (g.at(b, x, y, z) ? votes : 0) - c > 0;
  }
};
template <> struct Vote<kU8> {   // uint8 arithmetic: v * votes - count wraps modulo 256
  using T = uint8_t;
  static __device__ __forceinline__ bool keep(const Grid<T>& g, int64_t b, int x, int y, int z, int64_t votes, int c) {
    return (uint8_t)(g.at(b, x, y, z) * (uint8_t)votes - (uint8_t)c) != 0;
  }
};
template <> struct Vote<kF32> {
  using T = float;
  static __device__ __forceinline__ bool keep(const Grid<T>& g, int64_t b, int x, int y, int z, int64_t votes, int c) {
    return __fsub_rn(__fmul_rn(g.at(b, x, y, z), (float)votes), (float)c) > 0.f;
  }
};
template <> struct Vote<kF64> {
  using T = double;
  static __device__ __forceinline__ bool keep(const Grid<T>& g, int64_t b, int x, int y, int z, int64_t votes, int c) {
    return __dsub_rn(__dmul_rn(g.at(b, x, y, z), (double)votes), (double)c) > 0.0;
  }
};

template <typename O, int K>
__global__ void __launch_bounds__(kThreads) vg_project_kernel(const O* __restrict__ odms, Grid<typename Vote<K>::T> g,
                                                              int64_t B, int D, int64_t votes,
                                                              uint8_t* __restrict__ out) {
  using P = Odm<O>;
  const int64_t N = (int64_t)D * D * D, DD = (int64_t)D * D, total = B * N;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / N;
    const int v = (int)(i - b * N), x = v / (int)DD, y = (v / D) % D, z = v % D;
    const O* m = odms + b * 6 * DD;
    const int64_t xy = (int64_t)x * D + y, xz = (int64_t)x * D + z, yz = (int64_t)y * D + z;
    const int c = P::ge(z, P::rsub(D, m[xy])) + P::lt(z, m[DD + xy]) + P::ge(y, P::rsub(D, m[2 * DD + xz])) +
                  P::lt(y, m[3 * DD + xz]) + P::ge(x, P::rsub(D, m[4 * DD + yz])) + P::lt(x, m[5 * DD + yz]);
    out[i] = (uint8_t)Vote<K>::keep(g, b, x, y, z, votes, c);
  }
}

// ---------------------------------------------------------------------------------------------
// Host side.

// Sizes: batch, X, Y, Z >= 0 (else EINVAL) and X Y Z < 2^31 - 1 voxels per view (else ESIZE), with
// room for the fill's labels.
int vg_shape(int64_t batch, int64_t X, int64_t Y, int64_t Z, int64_t* N) {
  if (batch < 0 || X < 0 || Y < 0 || Z < 0) return DIBR_B200_EINVAL;
  *N = 0;
  if (X == 0 || Y == 0 || Z == 0) return 0;
  if (X >= INT32_MAX || Y >= INT32_MAX || Z >= INT32_MAX || X * Y >= INT32_MAX || X * Y * Z >= INT32_MAX)
    return DIBR_B200_ESIZE;
  *N = X * Y * Z;
  if (batch > (INT64_MAX / 8) / *N) return DIBR_B200_ESIZE;
  return 0;
}

template <typename T>
Grid<T> grid_of(const void* p, int64_t sb, int64_t sx, int64_t sy, int64_t sz) {
  return Grid<T>{(const T*)p, sb, sx, sy, sz};
}

template <typename T>
int vg_fill(const FillShape& s, Grid<T> g, int* L, uint8_t* out, cudaStream_t st) {
  {
    Span sp("vg_fill_init_kernel", st);
    vg_fill_init_kernel<T><<<grid_stride_ctas(32 * s.rows), kThreads, 0, st>>>(g, s, L);
  }
  {
    Span sp("vg_fill_merge_kernel", st);
    vg_fill_merge_kernel<<<grid_stride_ctas(32 * s.rows), kThreads, 0, st>>>(s, L);
  }
  Span sp("vg_fill_output_kernel", st);
  vg_fill_output_kernel<<<grid_stride_ctas((s.B * s.N + 15) / 16), kThreads, 0, st>>>(s, L, out);
  return (int)cudaGetLastError();
}

template <typename T, bool kThin>
int vg_surface(SurfShape s, Grid<T> g, uint8_t* out, cudaStream_t st) {
  Span sp(kThin ? "vg_surface_kernel<thin>" : "vg_surface_kernel<wide>", st);
  vg_surface_kernel<T, kThin><<<grid_stride_ctas(s.tiles, 1), dim3(kSurfZ, kSurfY), 0, st>>>(g, s, out);
  return (int)cudaGetLastError();
}

template <typename T>
int vg_odms(Grid<T> g, int64_t B, int D, int64_t* out, cudaStream_t st) {
  const int64_t n = B * 6 * (int64_t)D * D, t1 = (D + kOdmTile - 1) / kOdmTile;
  {
    Span sp("vg_odms_init_kernel", st);
    vg_odms_init_kernel<<<grid_stride_ctas(n), kThreads, 0, st>>>(n, D, (long long*)out);
  }
  Span sp("vg_odms_kernel", st);
  vg_odms_kernel<T><<<grid_stride_ctas(B * t1 * t1, 1), 32 * kOdmTile, 0, st>>>(g, B, D, (long long*)out);
  return (int)cudaGetLastError();
}

template <typename O, int K>
int vg_project(const void* odms, const void* grid, int64_t sb, int64_t sx, int64_t sy, int64_t sz, int64_t B, int D,
               int64_t votes, uint8_t* out, cudaStream_t st) {
  Span sp("vg_project_kernel", st);
  using T = typename Vote<K>::T;
  vg_project_kernel<O, K><<<grid_stride_ctas(B * (int64_t)D * D * D), kThreads, 0, st>>>(
      (const O*)odms, grid_of<T>(grid, sb, sx, sy, sz), B, D, votes, out);
  return (int)cudaGetLastError();
}

template <typename O>
int vg_project_grid(int grid_dtype, const void* odms, const void* grid, int64_t sb, int64_t sx, int64_t sy, int64_t sz,
                    int64_t B, int D, int64_t votes, uint8_t* out, cudaStream_t st) {
  switch (grid_dtype) {
    case DIBR_B200_VOXELGRID_ALL_ONES: return vg_project<O, kAllOnes>(odms, grid, sb, sx, sy, sz, B, D, votes, out, st);
    case DIBR_B200_DTYPE_BOOL: return vg_project<O, kBool>(odms, grid, sb, sx, sy, sz, B, D, votes, out, st);
    case DIBR_B200_DTYPE_U8: return vg_project<O, kU8>(odms, grid, sb, sx, sy, sz, B, D, votes, out, st);
    case DIBR_B200_DTYPE_F32: return vg_project<O, kF32>(odms, grid, sb, sx, sy, sz, B, D, votes, out, st);
    default: return vg_project<O, kF64>(odms, grid, sb, sx, sy, sz, B, D, votes, out, st);
  }
}

}  // namespace

int dibr_b200_voxelgrid_fill_workspace_bytes(int64_t batch, int64_t X, int64_t Y, int64_t Z,
                                             size_t* workspace_bytes) {
  if (!workspace_bytes) return DIBR_B200_EINVAL;
  int64_t N;
  if (const int e = vg_shape(batch, X, Y, Z, &N)) return e;
  *workspace_bytes = dibr_layout::voxelgrid_fill_layout(batch, N).bytes;
  return 0;
}

int dibr_b200_voxelgrid_fill(int64_t batch, int64_t X, int64_t Y, int64_t Z, int dtype, const void* grid,
                             int64_t stride_b, int64_t stride_x, int64_t stride_y, int64_t stride_z, uint8_t* out,
                             void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream) {
  int64_t N;
  if (const int e = vg_shape(batch, X, Y, Z, &N)) return e;
  if (dtype != DIBR_B200_DTYPE_F32 && dtype != DIBR_B200_DTYPE_U8) return DIBR_B200_EINVAL;
  if (batch * N == 0) return 0;
  if (!grid || !out || ((uintptr_t)out & 15)) return DIBR_B200_EINVAL;
  const dibr_layout::VoxelgridFillLayout Lo = dibr_layout::voxelgrid_fill_layout(batch, N);
  char* o = dibr_layout::carve(workspace, workspace_bytes, Lo.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  const FillShape s{batch, batch * X * Y, (int)X, (int)Y, (int)Z, (int)N};
  int* L = dibr_layout::piece<int>(o, Lo.labels);
  cudaStream_t st = (cudaStream_t)stream;
  return dtype == DIBR_B200_DTYPE_F32
             ? vg_fill(s, grid_of<float>(grid, stride_b, stride_x, stride_y, stride_z), L, out, st)
             : vg_fill(s, grid_of<uint8_t>(grid, stride_b, stride_x, stride_y, stride_z), L, out, st);
}

int dibr_b200_voxelgrid_extract_surface(int64_t batch, int64_t X, int64_t Y, int64_t Z, int dtype, int thin,
                                        const void* grid, int64_t stride_b, int64_t stride_x, int64_t stride_y,
                                        int64_t stride_z, uint8_t* out, dibr_b200_stream_t stream) {
  int64_t N;
  if (const int e = vg_shape(batch, X, Y, Z, &N)) return e;
  if (dtype != DIBR_B200_DTYPE_U8 && dtype != DIBR_B200_DTYPE_F32 && dtype != DIBR_B200_DTYPE_F64)
    return DIBR_B200_EINVAL;
  if (batch * N == 0) return 0;
  if (!grid || !out) return DIBR_B200_EINVAL;
  SurfShape s;
  s.B = batch; s.X = (int)X; s.Y = (int)Y; s.Z = (int)Z;
  s.tx = (int)((X + kSurfX - 1) / kSurfX); s.ty = (int)((Y + kSurfY - 1) / kSurfY); s.tz = (int)((Z + kSurfZ - 1) / kSurfZ);
  s.tiles = batch * s.tx * s.ty * s.tz;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t sb = stride_b, sx = stride_x, sy = stride_y, sz = stride_z;
  if (dtype == DIBR_B200_DTYPE_U8)
    return thin ? vg_surface<uint8_t, true>(s, grid_of<uint8_t>(grid, sb, sx, sy, sz), out, st)
                : vg_surface<uint8_t, false>(s, grid_of<uint8_t>(grid, sb, sx, sy, sz), out, st);
  if (dtype == DIBR_B200_DTYPE_F32)
    return thin ? vg_surface<float, true>(s, grid_of<float>(grid, sb, sx, sy, sz), out, st)
                : vg_surface<float, false>(s, grid_of<float>(grid, sb, sx, sy, sz), out, st);
  return thin ? vg_surface<double, true>(s, grid_of<double>(grid, sb, sx, sy, sz), out, st)
              : vg_surface<double, false>(s, grid_of<double>(grid, sb, sx, sy, sz), out, st);
}

int dibr_b200_voxelgrid_extract_odms(int64_t batch, int64_t dim, int dtype, const void* grid, int64_t stride_b,
                                     int64_t stride_x, int64_t stride_y, int64_t stride_z, int64_t* out,
                                     dibr_b200_stream_t stream) {
  int64_t N;
  if (const int e = vg_shape(batch, dim, dim, dim, &N)) return e;
  if (dtype != DIBR_B200_DTYPE_F32 && dtype != DIBR_B200_DTYPE_U8) return DIBR_B200_EINVAL;
  if (batch * N == 0) return 0;
  if (!grid || !out) return DIBR_B200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  return dtype == DIBR_B200_DTYPE_F32
             ? vg_odms(grid_of<float>(grid, stride_b, stride_x, stride_y, stride_z), batch, (int)dim, out, st)
             : vg_odms(grid_of<uint8_t>(grid, stride_b, stride_x, stride_y, stride_z), batch, (int)dim, out, st);
}

int dibr_b200_voxelgrid_project_odms(int64_t batch, int64_t dim, int odm_dtype, const void* odms, int grid_dtype,
                                     const void* grid, int64_t stride_b, int64_t stride_x, int64_t stride_y,
                                     int64_t stride_z, int64_t votes, uint8_t* out, dibr_b200_stream_t stream) {
  int64_t N;
  if (const int e = vg_shape(batch, dim, dim, dim, &N)) return e;
  if (odm_dtype != DIBR_B200_DTYPE_I64 && odm_dtype != DIBR_B200_DTYPE_I32 && odm_dtype != DIBR_B200_DTYPE_F32 &&
      odm_dtype != DIBR_B200_DTYPE_F64)
    return DIBR_B200_EINVAL;
  if (grid_dtype != DIBR_B200_VOXELGRID_ALL_ONES && grid_dtype != DIBR_B200_DTYPE_BOOL && grid_dtype != DIBR_B200_DTYPE_U8 &&
      grid_dtype != DIBR_B200_DTYPE_F32 && grid_dtype != DIBR_B200_DTYPE_F64)
    return DIBR_B200_EINVAL;
  if (batch * N == 0) return 0;
  if (!odms || !out || (grid_dtype != DIBR_B200_VOXELGRID_ALL_ONES && !grid)) return DIBR_B200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const int D = (int)dim;
  switch (odm_dtype) {
    case DIBR_B200_DTYPE_I64:
      return vg_project_grid<int64_t>(grid_dtype, odms, grid, stride_b, stride_x, stride_y, stride_z, batch, D, votes,
                                      out, st);
    case DIBR_B200_DTYPE_I32:
      return vg_project_grid<int32_t>(grid_dtype, odms, grid, stride_b, stride_x, stride_y, stride_z, batch, D, votes,
                                      out, st);
    case DIBR_B200_DTYPE_F32:
      return vg_project_grid<float>(grid_dtype, odms, grid, stride_b, stride_x, stride_y, stride_z, batch, D, votes,
                                    out, st);
    default:
      return vg_project_grid<double>(grid_dtype, odms, grid, stride_b, stride_x, stride_y, stride_z, batch, D, votes,
                                     out, st);
  }
}
