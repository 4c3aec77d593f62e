// mesh_topology.cu — the mesh Laplacian and vertex averaging of kaolin.ops.mesh (adjacency_matrix,
// uniform_laplacian, average_face_vertex_features / compute_vertex_normals) and
// kaolin.metrics.trianglemesh.uniform_laplacian_smoothing, behind the C ABI of include/dibr_b200.h.
//
// The reference builds a dense V x V matrix; here the topology of `faces` (F, S) is built once into
// two CSR structures in caller-owned buffers, O(F*S + V) in size:
//
//   corner CSR     for each vertex, the corners f*S + k that reference it, ordered by the key k*F + f
//                  (the order of the reference's `for k in range(S): scatter_add_` loop on the CPU)
//   adjacency CSR  for each vertex, its unique neighbours faces[f, (k +- 1) mod S] in ascending order
//                  (self-loops of degenerate faces included), its degree and fl(1 / degree)
//
// Build: count corners per vertex -> exclusive scan -> fill (atomic cursors, so in any order) ->
// sort and deduplicate every row (one thread per short row, one CTA per long row with an in-place
// bitonic network, so any row length works) -> scan of the degrees -> compaction.  The per-row sort
// makes the result independent of the order of the atomics: the build is deterministic.
//
// Every per-step kernel is a gather over one of the CSRs: no atomics, bit-reproducible.
//
// The same build serves Loop subdivision (triangle meshes) and, with all other corners of a cell as
// each corner's neighbours, tet meshes: marching tetrahedra and subdivide_tetmesh (end of the file).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dibr_b200.h"
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
using dibr_b200_detail::kScanTile;
using dibr_layout::carve;
using dibr_layout::piece;

constexpr int kScanThreads = 1024;
static_assert(kScanTile == kScanThreads * 4, "scan_*_kernel: four elements per thread");
constexpr int kShortRow = 32;                 // rows of at most this many corners are sorted by one thread
constexpr int kLongCtas = 132;                // CTAs that share out the long rows
constexpr int kThreads = 256;

inline unsigned grid_for(int64_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// Exclusive scan of one value per thread across the CTA (blockDim.x a multiple of 32); *total gets the sum.
__device__ int block_exclusive_scan(int v, int* total) {
  __shared__ int warp_sums[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int y = lane < nwarps ? warp_sums[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int z = __shfl_up_sync(0xffffffffu, y, o);
      if (lane >= o) y += z;
    }
    warp_sums[lane] = y;
  }
  __syncthreads();
  const int excl = x - v + (warp ? warp_sums[warp - 1] : 0);
  *total = warp_sums[nwarps - 1];
  __syncthreads();
  return excl;
}

// ---------------------------------------------------------------------------------------------
// Exclusive scan in[n] -> out[n + 1] (out[n] = the total) in three kernels: per-tile sums, a scan of
// the tile sums in one CTA, and the per-tile scan plus the tile's offset.
__global__ void __launch_bounds__(kScanThreads) scan_reduce_kernel(const int* __restrict__ in, int n,
                                                                   int* __restrict__ sums) {
  const int64_t base = (int64_t)blockIdx.x * kScanTile + 4 * threadIdx.x;
  int s = 0;
#pragma unroll
  for (int u = 0; u < 4; ++u)
    if (base + u < n) s += in[base + u];
  int total;
  block_exclusive_scan(s, &total);
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanThreads) scan_tiles_kernel(int* __restrict__ sums, int tiles) {
  int carry = 0;
  for (int base = 0; base < tiles; base += kScanThreads) {
    const int i = base + threadIdx.x;
    const int v = i < tiles ? sums[i] : 0;
    int total;
    const int excl = block_exclusive_scan(v, &total);
    if (i < tiles) sums[i] = carry + excl;
    carry += total;
  }
}

__global__ void __launch_bounds__(kScanThreads) scan_apply_kernel(const int* __restrict__ in, int n,
                                                                  const int* __restrict__ sums,
                                                                  int* __restrict__ out) {
  const int64_t base = (int64_t)blockIdx.x * kScanTile + 4 * threadIdx.x;
  int v[4], s = 0;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    v[u] = base + u < n ? in[base + u] : 0;
    s += v[u];
  }
  int total;
  int run = sums[blockIdx.x] + block_exclusive_scan(s, &total);
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    if (base + u < n) out[base + u] = run;
    run += v[u];
    if (base + u == n - 1) out[n] = run;
  }
}

}  // namespace

int dibr_b200_detail::exclusive_scan(const int* in, int n, int* sums, int* out, cudaStream_t st) {
  if (n == 0) return (int)cudaMemsetAsync(out, 0, sizeof(int), st);
  const int tiles = (int)((n + kScanTile - 1) / kScanTile);
  { Span s("scan_reduce_kernel", st); scan_reduce_kernel<<<tiles, kScanThreads, 0, st>>>(in, n, sums); }
  { Span s("scan_tiles_kernel", st); scan_tiles_kernel<<<1, kScanThreads, 0, st>>>(sums, tiles); }
  { Span s("scan_apply_kernel", st); scan_apply_kernel<<<tiles, kScanThreads, 0, st>>>(in, n, sums, out); }
  return (int)cudaGetLastError();
}

namespace {

// ---------------------------------------------------------------------------------------------
// Build.
struct Topo {
  int V, S;
  int R;              // raw neighbours per corner: 2 (faces: the cyclic ones) or S - 1 (cells: all others)
  int F;              // fits: R*F*S < 2^31 is checked on the host
  const int64_t* faces;
  int* corner_ptr; int* corners; int* adj_ptr; int* adj; int* degree; float* weight; int* status;
  int* count; int* raw; int* sums; int* long_rows; int* long_count;
};

__device__ __forceinline__ bool valid_vertex(int64_t v, int V) { return v >= 0 && v < V; }

__global__ void __launch_bounds__(kThreads) topo_count_kernel(Topo t) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= (int64_t)t.F * t.S) return;
  const int64_t v = t.faces[c];
  if (!valid_vertex(v, t.V)) { atomicOr(t.status + 1, 1); return; }
  atomicAdd(t.count + v, 1);
}

// Each corner takes a slot of its vertex's row (in whatever order the atomics give) and writes its key
// and its R raw neighbours (R = 2: the cyclic ones, faces[f, k +- 1]; otherwise every other corner of
// the cell); the row sort below puts them in order.  Corners with an index outside [0, V) were counted
// nowhere and write nothing.
__global__ void __launch_bounds__(kThreads) topo_fill_kernel(Topo t) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= (int64_t)t.F * t.S) return;
  const int64_t v = t.faces[c];
  if (!valid_vertex(v, t.V)) return;
  const int f = (int)(c / t.S), k = (int)(c - (int64_t)f * t.S);
  const int p = t.corner_ptr[v] + atomicSub(t.count + v, 1) - 1;
  t.corners[p] = k * t.F + f;
  const int64_t* row = t.faces + (int64_t)f * t.S;
  int* out = t.raw + (int64_t)t.R * p;
  if (t.R == 2) {
    out[0] = (int)row[k + 1 == t.S ? 0 : k + 1];
    out[1] = (int)row[k == 0 ? t.S - 1 : k - 1];
  } else {
    for (int u = 0, m = 0; u < t.S; ++u)
      if (u != k) out[m++] = (int)row[u];
  }
}

__device__ __forceinline__ void finish_row(const Topo& t, int v, int unique) {
  t.degree[v] = unique;
  t.weight[v] = unique ? 1.0f / (float)unique : 0.0f;   // IEEE division: torch.div(A, num_neighbour)
}

// Keys k*F + f -> corner ids f*S + k, in the same (key) order.
__device__ __forceinline__ int key_to_corner(int key, int F, int S) {
  const int k = key / F, f = key - k * F;
  return f * S + k;
}

// One thread per row of at most kShortRow corners; longer rows are listed for topo_sort_long_kernel.
__global__ void __launch_bounds__(kThreads) topo_sort_rows_kernel(Topo t) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= t.V) return;
  const int b = t.corner_ptr[v], n = t.corner_ptr[v + 1] - b;
  if (n > kShortRow) {
    t.long_rows[atomicAdd(t.long_count, 1)] = v;
    return;
  }
  int* keys = t.corners + b;
  insertion_sort(keys, n);
  for (int i = 0; i < n; ++i) keys[i] = key_to_corner(keys[i], t.F, t.S);
  int* nb = t.raw + (int64_t)t.R * b;
  insertion_sort(nb, t.R * n);
  int u = 0;
  for (int i = 0; i < t.R * n; ++i)
    if (i == 0 || nb[i] != nb[u - 1]) nb[u++] = nb[i];
  finish_row(t, v, u);
}

__global__ void __launch_bounds__(kScanThreads) topo_sort_long_kernel(Topo t) {
  __shared__ int last;
  const int rows = *t.long_count;
  for (int r = blockIdx.x; r < rows; r += gridDim.x) {
    const int v = t.long_rows[r];
    const int b = t.corner_ptr[v], n = t.corner_ptr[v + 1] - b;
    int* keys = t.corners + b;
    block_bitonic_sort(keys, n);
    for (int i = threadIdx.x; i < n; i += blockDim.x) keys[i] = key_to_corner(keys[i], t.F, t.S);
    int* nb = t.raw + (int64_t)t.R * b;
    const int m = t.R * n;
    block_bitonic_sort(nb, m);
    // in-place deduplication: chunk by chunk, each thread reads its value and its predecessor before
    // any write of the chunk; writes land at or below the chunk's first index, so only the value
    // before the chunk can have been overwritten, and it is kept in `last`
    int carry = 0;
    for (int base = 0; base < m; base += blockDim.x) {
      const int i = base + threadIdx.x;
      const int x = i < m ? nb[i] : 0;
      const int prev = i == 0 ? 0 : threadIdx.x == 0 ? last : (i < m ? nb[i - 1] : 0);
      const int keep = i < m && (i == 0 || x != prev);
      int total;
      const int pos = block_exclusive_scan(keep, &total);   // its barriers order the reads before the writes
      if (keep) nb[carry + pos] = x;
      if (i == base + (int)blockDim.x - 1 || i == m - 1) last = x;
      carry += total;
      __syncthreads();
    }
    if (threadIdx.x == 0) finish_row(t, v, carry);
    __syncthreads();
  }
}

// One warp per row: the row's unique neighbours move from the raw layout to the adjacency CSR.
__global__ void __launch_bounds__(kThreads) topo_compact_kernel(Topo t) {
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w == 0 && lane == 0) t.status[0] = t.adj_ptr[t.V];
  if (w >= t.V) return;
  const int v = (int)w;
  const int* src = t.raw + (int64_t)t.R * t.corner_ptr[v];
  const int b = t.adj_ptr[v], n = t.adj_ptr[v + 1] - b;
  for (int i = lane; i < n; i += 32) t.adj[b + i] = src[i];
}

// 0, or the error: V must leave room for V + 1 offsets, and the R*F*S raw neighbour entries (so
// every offset and every key k*F + f) must fit a 32-bit int.
int topo_dims(int V, int64_t F, int S, int R = 2) {
  if (V < 0 || F < 0 || S < 3) return DIBR_B200_EINVAL;
  if (V == INT32_MAX || F > (int64_t)INT32_MAX / S / R) return DIBR_B200_ESIZE;
  return 0;
}

// The build of both CSRs, with the pieces l at the workspace origin o; arguments checked by the caller.
int topo_build(Topo& t, char* o, const dibr_layout::TopoPieces& l, cudaStream_t st) {
  t.count = piece<int>(o, l.count); t.raw = piece<int>(o, l.raw); t.sums = piece<int>(o, l.sums);
  t.long_rows = piece<int>(o, l.long_rows); t.long_count = piece<int>(o, l.long_count);
  const int V = t.V;
  const int64_t FS = (int64_t)t.F * t.S;
  if (cudaMemsetAsync(t.status, 0, 2 * sizeof(int), st) != cudaSuccess) return (int)cudaGetLastError();
  if (V > 0 && cudaMemsetAsync(t.count, 0, sizeof(int) * (size_t)V, st) != cudaSuccess) return (int)cudaGetLastError();
  if (cudaMemsetAsync(t.long_count, 0, sizeof(int), st) != cudaSuccess) return (int)cudaGetLastError();
  if (FS > 0) { Span s("topo_count_kernel", st); topo_count_kernel<<<grid_for(FS, kThreads), kThreads, 0, st>>>(t); }
  if (int e = exclusive_scan(t.count, V, t.sums, t.corner_ptr, st)) return e;
  if (FS > 0) { Span s("topo_fill_kernel", st); topo_fill_kernel<<<grid_for(FS, kThreads), kThreads, 0, st>>>(t); }
  if (V > 0) {
    { Span s("topo_sort_rows_kernel", st); topo_sort_rows_kernel<<<grid_for(V, kThreads), kThreads, 0, st>>>(t); }
    { Span s("topo_sort_long_kernel", st); topo_sort_long_kernel<<<kLongCtas, kScanThreads, 0, st>>>(t); }
  }
  if (int e = exclusive_scan(t.degree, V, t.sums, t.adj_ptr, st)) return e;
  {
    Span s("topo_compact_kernel", st);
    topo_compact_kernel<<<grid_for(32 * (int64_t)(V > 0 ? V : 1), kThreads), kThreads, 0, st>>>(t);
  }
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Per-step kernels.

// y = L x (TRANSPOSE: L^T x), SMOOTH: (L + I) x, for x (B, V, 3): one thread per (view, vertex).
//   L x:    y_i = w_i sum_{j in N(i), j != i} x_j - x_i
//   L^T x:  y_j = sum_{i in N(j), i != j} w_i x_i - x_j    (the adjacency is symmetric)
template <bool TRANSPOSE, bool SMOOTH>
__global__ void __launch_bounds__(kThreads) laplacian_apply3_kernel(int64_t rows, int V, const int* __restrict__ adj_ptr,
                                                                    const int* __restrict__ adj,
                                                                    const float* __restrict__ weight,
                                                                    const float* __restrict__ x, float* __restrict__ y) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int i = (int)(r % V);
  const float* xb = x + (r - i) * 3;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
  const int e1 = __ldg(adj_ptr + i + 1);
  for (int e = __ldg(adj_ptr + i); e < e1; ++e) {
    const int j = __ldg(adj + e);
    if (j == i) continue;
    const float w = TRANSPOSE ? __ldg(weight + j) : 1.0f;
    const float* xj = xb + 3 * (int64_t)j;
    if (TRANSPOSE) {
      s0 += w * __ldg(xj); s1 += w * __ldg(xj + 1); s2 += w * __ldg(xj + 2);
    } else {
      s0 += __ldg(xj); s1 += __ldg(xj + 1); s2 += __ldg(xj + 2);
    }
  }
  if (!TRANSPOSE) {
    const float w = __ldg(weight + i);
    s0 = w * s0; s1 = w * s1; s2 = w * s2;
  }
  float* yr = y + 3 * r;
  if (SMOOTH) {
    yr[0] = s0; yr[1] = s1; yr[2] = s2;
  } else {
    const float* xi = x + 3 * r;
    yr[0] = s0 - __ldg(xi); yr[1] = s1 - __ldg(xi + 1); yr[2] = s2 - __ldg(xi + 2);
  }
}

// The same for any channel count C: one thread per (view, vertex, channel).
template <bool TRANSPOSE, bool SMOOTH>
__global__ void __launch_bounds__(kThreads) laplacian_apply_kernel(int64_t total, int V, int C, const int* __restrict__ adj_ptr,
                                                                   const int* __restrict__ adj,
                                                                   const float* __restrict__ weight,
                                                                   const float* __restrict__ x, float* __restrict__ y) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int64_t r = t / C;
  const int c = (int)(t - r * C);
  const int i = (int)(r % V);
  const float* xb = x + (r - i) * C + c;
  float s = 0.f;
  const int e1 = __ldg(adj_ptr + i + 1);
  for (int e = __ldg(adj_ptr + i); e < e1; ++e) {
    const int j = __ldg(adj + e);
    if (j == i) continue;
    const float v = __ldg(xb + (int64_t)j * C);
    s += TRANSPOSE ? __ldg(weight + j) * v : v;
  }
  if (!TRANSPOSE) s = __ldg(weight + i) * s;
  y[t] = SMOOTH ? s : s - __ldg(x + t);
}

// out[b, v, c] = (sum over v's corners in key order of ff[b, corner, c]) / max(count, 1)
__global__ void __launch_bounds__(kThreads) vertex_average_kernel(int64_t total, int V, int64_t FS, int C,
                                                                  const int* __restrict__ corner_ptr,
                                                                  const int* __restrict__ corners,
                                                                  const float* __restrict__ ff, float* __restrict__ out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int64_t r = t / C;
  const int c = (int)(t - r * C);
  const int64_t b = r / V;
  const int v = (int)(r - b * V);
  const float* src = ff + b * FS * C + c;
  const int p0 = __ldg(corner_ptr + v), p1 = __ldg(corner_ptr + v + 1);
  float s = 0.f;
  for (int p = p0; p < p1; ++p) s += __ldg(src + (int64_t)__ldg(corners + p) * C);
  const int n = p1 - p0;
  out[t] = s / (float)(n > 1 ? n : 1);
}

// grad_ff[b, f, k, c] = grad_out[b, faces[f, k], c] / max(count, 1)
__global__ void __launch_bounds__(kThreads) vertex_average_bwd_kernel(int64_t total, int V, int64_t FS, int C,
                                                                      const int64_t* __restrict__ faces,
                                                                      const int* __restrict__ corner_ptr,
                                                                      const float* __restrict__ g, float* __restrict__ gff) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int64_t r = t / C;
  const int c = (int)(t - r * C);
  const int64_t b = r / FS;
  const int v = (int)__ldg(faces + (r - b * FS));
  const int n = __ldg(corner_ptr + v + 1) - __ldg(corner_ptr + v);
  gff[t] = __ldg(g + (b * V + v) * C + c) / (float)(n > 1 ? n : 1);
}

// Dense (V, V): LAPLACIAN: -1 on the diagonal, w_i at the neighbours, 0 elsewhere; otherwise 1 at the
// neighbours (self-loops included) and 0 elsewhere.  Every element is written.
template <bool LAPLACIAN>
__global__ void __launch_bounds__(kThreads) dense_kernel(int V, const int* __restrict__ adj_ptr, const int* __restrict__ adj,
                                                         const float* __restrict__ weight, float* __restrict__ out) {
  const int64_t n = (int64_t)V * V;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(t / V), j = (int)(t - (int64_t)i * V);
    int lo = __ldg(adj_ptr + i), hi = __ldg(adj_ptr + i + 1);
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (__ldg(adj + mid) < j) lo = mid + 1; else hi = mid;
    }
    const bool hit = lo < __ldg(adj_ptr + i + 1) && __ldg(adj + lo) == j;
    float v;
    if (LAPLACIAN) v = i == j ? -1.0f : hit ? __ldg(weight + i) : 0.0f;
    else v = hit ? 1.0f : 0.0f;
    out[t] = v;
  }
}

// COO indices (2, E) of the adjacency, rows and columns in CSR (row-major) order: one warp per row.
__global__ void __launch_bounds__(kThreads) adjacency_coo_kernel(int V, int64_t E, const int* __restrict__ adj_ptr,
                                                                 const int* __restrict__ adj, int64_t* __restrict__ idx) {
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= V) return;
  const int b = adj_ptr[w], e = adj_ptr[w + 1];
  for (int i = b + lane; i < e; i += 32) {
    idx[i] = w;
    idx[E + i] = adj[i];
  }
}

// ---------------------------------------------------------------------------------------------
// Loop subdivision (kaolin.ops.mesh.subdivide_trianglemesh), one level on top of the topology of a
// triangle mesh.  The reference's unique edges, in lexicographic order, are the adjacency entries
// (i, j) with j >= i in CSR order, so edge ids are a scan over rows of the number of such entries:
// the entry at position p of row a has the id p + edge_ptr[a + 1] - adj_ptr[a + 1].  Edge e becomes
// vertex V + e; edges[e] = {a, b, f0, f1} with a <= b, and f0 <= f1 the faces of its two face edges
// when it has exactly two, f0 = f1 = -1 for any other count.
struct Subdiv {
  int V, F;
  const int64_t* faces;
  const int* corner_ptr; const int* corners; const int* adj_ptr; const int* adj;
  int* count; int* edge_ptr; int* adj_edge; int* face_edge; int4* edges; int64_t* new_faces;
  int2* pairs;        // tet meshes: {a, b} per edge instead of the face record
};

__device__ __forceinline__ int lower_bound_row(const int* __restrict__ adj, int lo, int hi, int key) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(adj + mid) < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// The id of edge (a, b), a <= b both in [0, V); -1 when b is not a neighbour of a.
__device__ __forceinline__ int edge_id(const Subdiv& s, int a, int b) {
  const int e1 = __ldg(s.adj_ptr + a + 1);
  const int p = lower_bound_row(s.adj, __ldg(s.adj_ptr + a), e1, b);
  return p < e1 && __ldg(s.adj + p) == b ? p + s.edge_ptr[a + 1] - e1 : -1;
}

// count[i] = the number of neighbours j >= i of row i.
__global__ void __launch_bounds__(kThreads) subdiv_count_kernel(Subdiv s) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= s.V) return;
  const int e1 = __ldg(s.adj_ptr + i + 1);
  s.count[i] = e1 - lower_bound_row(s.adj, __ldg(s.adj_ptr + i), e1, i);
}

// One thread per adjacency entry (i, j): its edge id, and for j >= i the edge record: FACES (triangle
// meshes) the int4 record with the edge's two faces, otherwise (tet meshes) the pair {i, j}.  The face
// edges (f, k) of edge (i, j) are found among the corners of i: corner k of f starts face edge k, whose
// other end is faces[f, k+1], and ends face edge k-1, whose other end is faces[f, k-1] (counted there
// only when j != i, so that a self-loop's face edge is counted once).  Entries naming a vertex outside
// [0, V) exist only when the topology build reported an error; they get id -1.
template <bool FACES>
__global__ void __launch_bounds__(kThreads) subdiv_edges_kernel(Subdiv s, int64_t capacity) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= capacity) return;
  const int p = (int)q, V = s.V;
  if (p >= __ldg(s.adj_ptr + V)) return;
  int lo = 0, hi = V + 1;                       // the row of p: the last i with adj_ptr[i] <= p
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(s.adj_ptr + mid) <= p) lo = mid + 1; else hi = mid;
  }
  const int i = lo - 1, j = __ldg(s.adj + p);
  if (!valid_vertex(j, V)) { s.adj_edge[p] = -1; return; }
  if (j < i) { s.adj_edge[p] = edge_id(s, j, i); return; }
  const int id = p + s.edge_ptr[i + 1] - __ldg(s.adj_ptr + i + 1);
  s.adj_edge[p] = id;
  if (!FACES) { s.pairs[id] = make_int2(i, j); return; }
  int n = 0, f0 = -1, f1 = -1;
  for (int c = __ldg(s.corner_ptr + i), c1 = __ldg(s.corner_ptr + i + 1); c < c1; ++c) {
    const int corner = __ldg(s.corners + c), f = corner / 3, k = corner - 3 * f;
    const int64_t* row = s.faces + 3 * (int64_t)f;
    const int m = (__ldg(row + (k == 2 ? 0 : k + 1)) == j) + (j != i && __ldg(row + (k == 0 ? 2 : k - 1)) == j);
    for (int u = 0; u < m; ++u, ++n) {
      if (n == 0) f0 = f;
      else if (n == 1) f1 = f;
    }
  }
  if (n != 2) f0 = f1 = -1;
  else if (f1 < f0) { const int t = f0; f0 = f1; f1 = t; }
  s.edges[id] = make_int4(i, j, f0, f1);
}

// One thread per face: the ids of its edges (f0,f1), (f1,f2), (f2,f0) and its four child faces
// (v0, v1, v2, V+e01, V+e12, V+e20)[[1,4,3], [0,3,5], [2,5,4], [5,3,4]].
__global__ void __launch_bounds__(kThreads) subdiv_faces_kernel(Subdiv s) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= s.F) return;
  const int64_t* row = s.faces + 3 * (int64_t)f;
  int64_t v[6];
#pragma unroll
  for (int k = 0; k < 3; ++k) v[k] = __ldg(row + k);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int64_t a = v[k] < v[k == 2 ? 0 : k + 1] ? v[k] : v[k == 2 ? 0 : k + 1];
    const int64_t b = v[k] < v[k == 2 ? 0 : k + 1] ? v[k == 2 ? 0 : k + 1] : v[k];
    const int e = valid_vertex(a, s.V) && valid_vertex(b, s.V) ? edge_id(s, (int)a, (int)b) : -1;
    s.face_edge[3 * f + k] = e;
    v[3 + k] = (int64_t)s.V + e;
  }
  constexpr int kChild[12] = {1, 4, 3, 0, 3, 5, 2, 5, 4, 5, 3, 4};
  int64_t* out = s.new_faces + 12 * (int64_t)f;
#pragma unroll
  for (int u = 0; u < 12; ++u) out[u] = v[kChild[u]];
}

// The reference's default weight of a vertex of n neighbours, _get_alpha(n) * n, in its fp32 steps:
// torch evaluates 2*pi / n as reciprocal(n) * 2*pi.  n = 0 gives NaN.
__device__ __forceinline__ float default_alpha(int deg) {
  const float n = (float)deg;
  const float c = __fadd_rn(0.375f, __fmul_rn(0.25f, cosf(__fmul_rn(1.0f / n, 6.28318530717958648f))));
  const float a = deg == 3 ? 0.1875f : __fsub_rn(0.625f, __fmul_rn(c, c)) / n;
  return __fmul_rn(a, n);
}

// One thread per output vertex (view b, row r < V + E):
//   r < V  even:  (1 - a_r) x_r + (a_r / n_r) sum_{j in N(r)} x_j
//   r >= V odd, edge e = r - V = (a, b):  two faces: (sum of both faces' vertices + x_a + x_b) / 8,
//          otherwise (x_a + x_b) / 2.
// ALPHA: a is the given (B, V) alpha, and alpha_out (if not NULL) gets the next level's alpha: a_r for
// even rows, the odd stencil over a for odd rows.  Otherwise a is default_alpha(n).
template <bool ALPHA>
__global__ void __launch_bounds__(kThreads) subdiv_forward_kernel(int64_t total, int V, int E,
                                                                  const int* __restrict__ adj_ptr,
                                                                  const int* __restrict__ adj,
                                                                  const int4* __restrict__ edges,
                                                                  const int64_t* __restrict__ faces,
                                                                  const float* __restrict__ x,
                                                                  const float* __restrict__ alpha,
                                                                  float* __restrict__ y, float* __restrict__ alpha_out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int W = V + E;
  const int64_t b = t / W;
  const int r = (int)(t - b * W);
  const float* xb = x + b * V * 3;
  const float* ab = ALPHA ? alpha + b * V : nullptr;
  float o0, o1, o2, oa = 0.f;
  if (r < V) {
    const int p0 = __ldg(adj_ptr + r), p1 = __ldg(adj_ptr + r + 1);
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int p = p0; p < p1; ++p) {
      const float* xj = xb + 3 * (int64_t)__ldg(adj + p);
      s0 += __ldg(xj); s1 += __ldg(xj + 1); s2 += __ldg(xj + 2);
    }
    const float a = ALPHA ? __ldg(ab + r) : default_alpha(p1 - p0);
    const float w = a / (float)(p1 - p0), u = 1.0f - a;
    const float* xr = xb + 3 * (int64_t)r;
    o0 = u * __ldg(xr) + w * s0; o1 = u * __ldg(xr + 1) + w * s1; o2 = u * __ldg(xr + 2) + w * s2;
    oa = ALPHA ? a : 0.f;
  } else {
    const int4 e = __ldg(edges + (r - V));
    const float *xa = xb + 3 * (int64_t)e.x, *xe = xb + 3 * (int64_t)e.y;
    if (e.z < 0) {
      o0 = (__ldg(xa) + __ldg(xe)) * 0.5f; o1 = (__ldg(xa + 1) + __ldg(xe + 1)) * 0.5f;
      o2 = (__ldg(xa + 2) + __ldg(xe + 2)) * 0.5f;
      if (ALPHA) oa = (__ldg(ab + e.x) + __ldg(ab + e.y)) * 0.5f;
    } else {
      int64_t v[8];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        v[k] = __ldg(faces + 3 * (int64_t)e.z + k);
        v[3 + k] = __ldg(faces + 3 * (int64_t)e.w + k);
      }
      v[6] = e.x; v[7] = e.y;
      o0 = o1 = o2 = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float* xv = xb + 3 * v[k];
        o0 += __ldg(xv); o1 += __ldg(xv + 1); o2 += __ldg(xv + 2);
        if (ALPHA) oa += __ldg(ab + v[k]);
      }
      o0 *= 0.125f; o1 *= 0.125f; o2 *= 0.125f; oa *= 0.125f;
    }
  }
  float* yr = y + 3 * t;
  yr[0] = o0; yr[1] = o1; yr[2] = o2;
  if (ALPHA && alpha_out) alpha_out[t] = oa;
}

// One thread per input vertex (view b, row j): the transpose of the forward, as a gather.
//   even self term   (1 - a_j) g_j
//   even neighbours  sum_{i in N(j)} (a_i / n_i) g_i               (the adjacency is symmetric)
//   edge endpoints   for each entry (j, i): w g_{V+e}, w = 1/8 (two faces) or 1/2, twice for i == j
//   face terms       for each corner of j in face f, each face edge of f with two faces: 1/8 g_{V+e}
// ALPHA (given alpha): grad_alpha_j = (g_j . s_j) / n_j - g_j . x_j (in fp64, then rounded), plus the
// carried alpha's gradient ga_j and the same endpoint and face terms over ga_{V+e}.
template <bool ALPHA>
__global__ void __launch_bounds__(kThreads) subdiv_backward_kernel(
    int64_t total, int V, int E, const int* __restrict__ corner_ptr, const int* __restrict__ corners,
    const int* __restrict__ adj_ptr, const int* __restrict__ adj, const int* __restrict__ adj_edge,
    const int* __restrict__ face_edge, const int4* __restrict__ edges, const float* __restrict__ x,
    const float* __restrict__ alpha, const float* __restrict__ gy, const float* __restrict__ gao,
    float* __restrict__ gx, float* __restrict__ ga) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int64_t b = t / V;
  const int j = (int)(t - b * V), W = V + E;
  const float* gyb = gy + b * W * 3;
  const float* gab = ALPHA && gao ? gao + b * W : nullptr;
  const float* xb = x + b * V * 3;
  const float* ab = ALPHA ? alpha + b * V : nullptr;
  const int* edge_two = reinterpret_cast<const int*>(edges) + 2;      // f0 of edge e at edge_two[4 e]
  const bool want_ga = ALPHA && ga;
  const int p0 = __ldg(adj_ptr + j), p1 = __ldg(adj_ptr + j + 1);
  const float* gj = gyb + 3 * (int64_t)j;
  const float gj0 = __ldg(gj), gj1 = __ldg(gj + 1), gj2 = __ldg(gj + 2);
  float n0 = 0.f, n1 = 0.f, n2 = 0.f;      // even neighbour terms
  float e0 = 0.f, e1 = 0.f, e2 = 0.f, ea = 0.f;   // edge terms
  // sum of the neighbours, for grad_alpha, in fp64: (g . s) / n and g . x nearly cancel on a smooth
  // surface, and the reference's CPU reductions accumulate in double
  double s0 = 0.0, s1 = 0.0, s2 = 0.0;
  for (int p = p0; p < p1; ++p) {
    const int i = __ldg(adj + p);
    const int q0 = __ldg(adj_ptr + i), q1 = __ldg(adj_ptr + i + 1);
    const float wi = (ALPHA ? __ldg(ab + i) : default_alpha(q1 - q0)) / (float)(q1 - q0);
    const float* gi = gyb + 3 * (int64_t)i;
    n0 += wi * __ldg(gi); n1 += wi * __ldg(gi + 1); n2 += wi * __ldg(gi + 2);
    if (want_ga) {
      const float* xi = xb + 3 * (int64_t)i;
      s0 += __ldg(xi); s1 += __ldg(xi + 1); s2 += __ldg(xi + 2);
    }
    const int e = __ldg(adj_edge + p);
    float w = __ldg(edge_two + 4 * (int64_t)e) < 0 ? 0.5f : 0.125f;
    if (i == j) w += w;
    const float* ge = gyb + 3 * ((int64_t)V + e);
    e0 += w * __ldg(ge); e1 += w * __ldg(ge + 1); e2 += w * __ldg(ge + 2);
    if (gab) ea += w * __ldg(gab + V + e);
  }
  for (int c = __ldg(corner_ptr + j), c1 = __ldg(corner_ptr + j + 1); c < c1; ++c) {
    const int* fe = face_edge + 3 * (__ldg(corners + c) / 3);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int e = __ldg(fe + k);
      if (__ldg(edge_two + 4 * (int64_t)e) < 0) continue;
      const float* ge = gyb + 3 * ((int64_t)V + e);
      e0 += 0.125f * __ldg(ge); e1 += 0.125f * __ldg(ge + 1); e2 += 0.125f * __ldg(ge + 2);
      if (gab) ea += 0.125f * __ldg(gab + V + e);
    }
  }
  const float aj = ALPHA ? __ldg(ab + j) : default_alpha(p1 - p0);
  if (gx) {
    const float u = 1.0f - aj;
    float* o = gx + 3 * t;
    o[0] = u * gj0 + n0 + e0; o[1] = u * gj1 + n1 + e1; o[2] = u * gj2 + n2 + e2;
  }
  if (want_ga) {
    const float* xj = xb + 3 * (int64_t)j;
    const double gs = (double)gj0 * s0 + (double)gj1 * s1 + (double)gj2 * s2;
    const double gv = (double)gj0 * __ldg(xj) + (double)gj1 * __ldg(xj + 1) + (double)gj2 * __ldg(xj + 2);
    ga[t] = (float)(gs / (double)(p1 - p0) - gv) + (gab ? __ldg(gab + j) : 0.f) + ea;
  }
}

// ---------------------------------------------------------------------------------------------
// Tet meshes (kaolin.ops.conversions.marching_tetrahedra, kaolin.ops.mesh.subdivide_tetmesh).  The
// topology is that of the cells (T, 4) with all three other corners as each corner's neighbours, so
// the adjacency holds the six edges of every tet; edges are numbered as for Loop subdivision, and
// tet_edge (T, 6) holds each tet's corner pairs 01, 02, 03, 12, 13, 23 as edge ids.
__global__ void __launch_bounds__(kThreads) tet_edges_kernel(Subdiv s) {
  constexpr int kTetPairA[6] = {0, 0, 0, 1, 1, 2};
  constexpr int kTetPairB[6] = {1, 2, 3, 2, 3, 3};
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= s.F) return;
  const int64_t* row = s.faces + 4 * (int64_t)t;
  int64_t v[4];
  bool ok = true;
#pragma unroll
  for (int k = 0; k < 4; ++k) { v[k] = __ldg(row + k); ok = ok && valid_vertex(v[k], s.V); }
#pragma unroll
  for (int u = 0; u < 6; ++u) {
    const int64_t a = v[kTetPairA[u]], b = v[kTetPairB[u]];
    s.face_edge[6 * (int64_t)t + u] = ok ? edge_id(s, (int)(a < b ? a : b), (int)(a < b ? b : a)) : -1;
  }
}

// Marching tetrahedra.  occ(v) = sdf(v) > 0 (0 and NaN are outside).  A tet's case is
// c = sum_k occ(corner k) 2^k; it has one triangle when 1 or 3 corners are inside, two when 2 are.
// Its triangles, in the order the reference emits them: each is three corner pairs, each pair one
// hex byte "ij" (the edge between corners i and j); slots past the case's triangles are 0.  Every
// pair a case uses joins an inside and an outside corner, so it always has an output vertex.
#define DIBR_B200_MT_CASES                                                                                \
  {                                                                                                       \
    0x000000000000ull, 0x020103000000ull, 0x130112000000ull, 0x021303021213ull, 0x120223000000ull,         \
    0x031201032312ull, 0x021301022313ull, 0x130323000000ull, 0x132303000000ull, 0x130201132302ull,         \
    0x120301122303ull, 0x021223000000ull, 0x130203131202ull, 0x120113000000ull, 0x030102000000ull,         \
    0x000000000000ull                                                                                     \
  }
__constant__ uint64_t kMtCases[16] = DIBR_B200_MT_CASES;
const uint64_t kMtCasesHost[16] = DIBR_B200_MT_CASES;

// Pair k (0..5) of a case word -> the tet's edge slot (0..5: 01, 02, 03, 12, 13, 23).
__host__ __device__ __forceinline__ int mt_pair_slot(uint64_t word, int k, int* a = nullptr, int* b = nullptr) {
  const int byte = (int)(word >> (40 - 8 * k)) & 0xff, i = byte >> 4, j = byte & 15;
  if (a) { *a = i; *b = j; }
  return i + j - 1 + (i > 0);
}

__device__ __forceinline__ int mt_triangles(int c) {
  const int n = __popc(c);
  return n == 2 ? 2 : (n & 1);
}

struct MTets {
  int B, V, E, T;
  const int2* edges; const int64_t* tets; const int* tet_edge; const float* x; const float* sdf;
  int* flags; const int* scan; int* vid; float* out_v; int64_t* out_f; int64_t* out_tet;
};

__device__ __forceinline__ int mt_case(const MTets& m, int b, int t) {
  const int64_t* row = m.tets + 4 * (int64_t)t;
  const float* s = m.sdf + (int64_t)b * m.V;
  int c = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) c |= (__ldg(s + __ldg(row + k)) > 0.f) << k;
  return c;
}

// flags = [B*E sign-change flags | B*T one-triangle flags | B*T two-triangle flags], one thread each
// for the first B*E and the next B*T.
__global__ void __launch_bounds__(kThreads) mt_classify_kernel(MTets m) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t BE = (int64_t)m.B * m.E, BT = (int64_t)m.B * m.T;
  if (q < BE) {
    const int b = (int)(q / m.E);
    const int2 e = __ldg(m.edges + (q - (int64_t)b * m.E));
    const float* s = m.sdf + (int64_t)b * m.V;
    m.flags[q] = (__ldg(s + e.x) > 0.f) != (__ldg(s + e.y) > 0.f);
  } else if (q < BE + BT) {
    const int64_t r = q - BE;
    const int b = (int)(r / m.T);
    const int n = mt_triangles(mt_case(m, b, (int)(r - (int64_t)b * m.T)));
    m.flags[BE + r] = n == 1;
    m.flags[BE + BT + r] = n == 2;
  }
}

// counts[b] = {vertices, one-triangle tets, two-triangle tets} of view b, from the scan of the flags.
__global__ void __launch_bounds__(kThreads) mt_counts_kernel(MTets m, int* __restrict__ counts) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= m.B) return;
  const int64_t BE = (int64_t)m.B * m.E, BT = (int64_t)m.B * m.T, E = m.E, T = m.T;
  counts[3 * b] = m.scan[(b + 1) * E] - m.scan[b * E];
  counts[3 * b + 1] = m.scan[BE + (b + 1) * T] - m.scan[BE + b * T];
  counts[3 * b + 2] = m.scan[BE + BT + (b + 1) * T] - m.scan[BE + BT + b * T];
}

// One thread per (view, edge): a sign-change edge (a, b) gets the output row scan[q] (rows of all
// views in one array, view by view) and the vertex (x_a (-s_b) + x_b s_a) / (s_a + (-s_b)), rounded
// step by step as the reference's separate element-wise ops are; vid[q] is the row, or -1.
__global__ void __launch_bounds__(kThreads) mt_vertices_kernel(MTets m) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= (int64_t)m.B * m.E) return;
  const int row = __ldg(m.scan + q);
  if (__ldg(m.scan + q + 1) == row) { m.vid[q] = -1; return; }
  m.vid[q] = row;
  const int b = (int)(q / m.E);
  const int2 e = __ldg(m.edges + (q - (int64_t)b * m.E));
  const int64_t ia = (int64_t)b * m.V + e.x, ib = (int64_t)b * m.V + e.y;
  const float sa = __ldg(m.sdf + ia), nb = -__ldg(m.sdf + ib);
  const float den = __fadd_rn(sa, nb);
  float* o = m.out_v + 3 * (int64_t)row;
#pragma unroll
  for (int c = 0; c < 3; ++c)
    o[c] = __fdiv_rn(__fadd_rn(__fmul_rn(__ldg(m.x + 3 * ia + c), nb), __fmul_rn(__ldg(m.x + 3 * ib + c), sa)), den);
}

// One thread per (view, tet): its triangles at their rows.  In view b, the faces of one-triangle tets
// come first in tet order, then two per two-triangle tet; views follow each other in one array.
// Vertex ids are per view.
__global__ void __launch_bounds__(kThreads) mt_faces_kernel(MTets m) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t BE = (int64_t)m.B * m.E, BT = (int64_t)m.B * m.T;
  if (r >= BT) return;
  const int b = (int)(r / m.T), t = (int)(r - (int64_t)b * m.T);
  const int c = mt_case(m, b, t), n = mt_triangles(c);
  if (n == 0) return;
  const int* one = m.scan + BE;          // exclusive scan of the one-triangle flags (continued by the two-)
  const int* two = one + BT;
  const int64_t v0 = (int64_t)b * m.T;
  const int one0 = __ldg(one + v0) - __ldg(one), two0 = __ldg(two + v0) - __ldg(two);
  int64_t f = one0 + 2 * (int64_t)two0;  // the view's first face
  if (n == 1) f += __ldg(one + r) - __ldg(one + v0);
  else f += (__ldg(one + v0 + m.T) - __ldg(one + v0)) + 2 * (int64_t)(__ldg(two + r) - __ldg(two + v0));
  const uint64_t word = kMtCases[c];
  const int* te = m.tet_edge + 6 * (int64_t)t;
  const int* vid = m.vid + (int64_t)b * m.E;
  const int base = __ldg(m.scan + (int64_t)b * m.E);
  for (int k = 0; k < 3 * n; ++k) m.out_f[3 * f + k] = vid[__ldg(te + mt_pair_slot(word, k))] - base;
  if (m.out_tet) for (int k = 0; k < n; ++k) m.out_tet[f + k] = t;
}

// One thread per (view, vertex i): the gradients of its sign-change edges, read from grad_out at each
// edge's vertex row, summed over i's adjacency row.  For an edge (a, b), with n = -s_b,
// d = s_a + n, num = x_a n + x_b s_a and y = num / d, as the reference's autograd forms them:
//   gn = g / d,  gd = sum_c -g_c ((num_c / d) / d)
//   x_a: gn n    x_b: gn s_a    s_a: sum_c gn_c x_b,c + gd    s_b: -(sum_c gn_c x_a,c + gd)
__global__ void __launch_bounds__(kThreads) mt_backward_kernel(int64_t total, int V, int E, const int* __restrict__ adj_ptr,
                                                               const int* __restrict__ adj,
                                                               const int* __restrict__ adj_edge,
                                                               const float* __restrict__ x, const float* __restrict__ sdf,
                                                               const int* __restrict__ vid, const float* __restrict__ g,
                                                               float* __restrict__ gx, float* __restrict__ gs) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= total) return;
  const int64_t b = q / V;
  const int i = (int)(q - b * V);
  const float* xb = x + b * V * 3;
  const float* sb = sdf + b * V;
  const int* vb = vid + b * E;
  float o0 = 0.f, o1 = 0.f, o2 = 0.f, os = 0.f;
  for (int p = __ldg(adj_ptr + i), p1 = __ldg(adj_ptr + i + 1); p < p1; ++p) {
    const int row = __ldg(vb + __ldg(adj_edge + p));
    if (row < 0) continue;
    const int j = __ldg(adj + p);
    const bool first = i < j;               // i is the edge's endpoint a
    const int ia = first ? i : j, ib = first ? j : i;
    const float sa = __ldg(sb + ia), n = -__ldg(sb + ib);
    const float d = __fadd_rn(sa, n);
    float gn[3], xa[3], xe[3], gd = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      xa[c] = __ldg(xb + 3 * (int64_t)ia + c);
      xe[c] = __ldg(xb + 3 * (int64_t)ib + c);
      const float gc = __ldg(g + 3 * (int64_t)row + c);
      const float num = __fadd_rn(__fmul_rn(xa[c], n), __fmul_rn(xe[c], sa));
      gn[c] = __fdiv_rn(gc, d);
      gd = __fadd_rn(gd, __fmul_rn(-gc, __fdiv_rn(__fdiv_rn(num, d), d)));
    }
    if (first) {
      o0 += __fmul_rn(gn[0], n); o1 += __fmul_rn(gn[1], n); o2 += __fmul_rn(gn[2], n);
      os += __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(gn[0], xe[0]), __fmul_rn(gn[1], xe[1])), __fmul_rn(gn[2], xe[2])), gd);
    } else {
      o0 += __fmul_rn(gn[0], sa); o1 += __fmul_rn(gn[1], sa); o2 += __fmul_rn(gn[2], sa);
      os -= __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(gn[0], xa[0]), __fmul_rn(gn[1], xa[1])), __fmul_rn(gn[2], xa[2])), gd);
    }
  }
  if (gx) { gx[3 * q] = o0; gx[3 * q + 1] = o1; gx[3 * q + 2] = o2; }
  if (gs) gs[q] = os;
}

// subdivide_tetmesh: one thread per output row (view b, row r < V + E) of the positions (3 channels)
// and the features (D channels, if any): row r < V is vertex r, row V + e the midpoint of edge e,
// (y_a + y_b) * 0.5 (the reference's mean of two).
__global__ void __launch_bounds__(kThreads) tet_subdivide_forward_kernel(int64_t total, int V, int E, int D,
                                                                         const int2* __restrict__ edges,
                                                                         const float* __restrict__ x,
                                                                         const float* __restrict__ f,
                                                                         float* __restrict__ y, float* __restrict__ yf) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= total) return;
  const int W = V + E;
  const int64_t b = q / W;
  const int r = (int)(q - b * W);
  int a = r, c = r;
  if (r >= V) { const int2 e = __ldg(edges + (r - V)); a = e.x; c = e.y; }
  const int64_t ia = b * V + a, ic = b * V + c;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float u = __ldg(x + 3 * ia + k);
    y[3 * q + k] = r < V ? u : __fmul_rn(__fadd_rn(u, __ldg(x + 3 * ic + k)), 0.5f);
  }
  for (int k = 0; k < D; ++k) {
    const float u = __ldg(f + D * ia + k);
    yf[D * q + k] = r < V ? u : __fmul_rn(__fadd_rn(u, __ldg(f + D * ic + k)), 0.5f);
  }
}

// One thread per tet: its eight children, child k at row k*T + t, over the ten vertices
// (v0, v1, v2, v3, V+e01, V+e02, V+e03, V+e12, V+e13, V+e23): a corner tet at each corner, then
// four tets of the inner octahedron around its diagonal (e01, e23).
__global__ void __launch_bounds__(kThreads) tet_children_kernel(int V, int T, const int64_t* __restrict__ tets,
                                                                const int* __restrict__ tet_edge,
                                                                int64_t* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  int64_t v[10];
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = __ldg(tets + 4 * (int64_t)t + k);
#pragma unroll
  for (int k = 0; k < 6; ++k) v[4 + k] = (int64_t)V + __ldg(tet_edge + 6 * (int64_t)t + k);
  constexpr int kChild[32] = {0, 4, 5, 6,  1, 7, 4, 8,  2, 5, 7, 9,  3, 6, 9, 8,
                              4, 5, 6, 8,  4, 5, 8, 7,  9, 5, 8, 6,  9, 5, 7, 8};
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    int64_t* o = out + 4 * ((int64_t)k * T + t);
#pragma unroll
    for (int u = 0; u < 4; ++u) o[u] = v[kChild[4 * k + u]];
  }
}

// One thread per (view b, input vertex i): its own row's gradient plus half that of every edge row
// of i's adjacency row (a self-loop's row is all of i's: twice a half).
__global__ void __launch_bounds__(kThreads) tet_subdivide_backward_kernel(int64_t total, int V, int E, int D,
                                                                          const int* __restrict__ adj_ptr,
                                                                          const int* __restrict__ adj,
                                                                          const int* __restrict__ adj_edge,
                                                                          const float* __restrict__ gy,
                                                                          const float* __restrict__ gyf,
                                                                          float* __restrict__ gx, float* __restrict__ gf) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= total) return;
  const int64_t b = q / V;
  const int i = (int)(q - b * V);
  const int64_t own = b * (V + E) + i, edge0 = b * (V + E) + V;
  const int p0 = __ldg(adj_ptr + i), p1 = __ldg(adj_ptr + i + 1);
  if (gx) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int p = p0; p < p1; ++p) {
      const float w = __ldg(adj + p) == i ? 1.0f : 0.5f;
      const float* ge = gy + 3 * (edge0 + __ldg(adj_edge + p));
      s0 += w * __ldg(ge); s1 += w * __ldg(ge + 1); s2 += w * __ldg(ge + 2);
    }
    gx[3 * q] = __ldg(gy + 3 * own) + s0; gx[3 * q + 1] = __ldg(gy + 3 * own + 1) + s1;
    gx[3 * q + 2] = __ldg(gy + 3 * own + 2) + s2;
  }
  if (gf) {
    for (int k = 0; k < D; ++k) {
      float s = 0.f;
      for (int p = p0; p < p1; ++p)
        s += (__ldg(adj + p) == i ? 1.0f : 0.5f) * __ldg(gyf + D * (edge0 + __ldg(adj_edge + p)) + k);
      gf[D * q + k] = __ldg(gyf + D * own + k) + s;
    }
  }
}

}  // namespace

extern "C" {

size_t dibr_b200_mesh_topology_workspace_bytes(int num_vertices, int64_t num_faces, int face_size) {
  if (topo_dims(num_vertices, num_faces, face_size)) return 0;
  return dibr_layout::mesh_topology_layout(num_vertices, num_faces, face_size).bytes;
}

int dibr_b200_mesh_topology_build(int num_vertices, int64_t num_faces, int face_size, const int64_t* faces,
                                  int32_t* corner_ptr, int32_t* corners, int32_t* adj_ptr, int32_t* adj,
                                  int32_t* degree, float* weight, int32_t* status, void* workspace,
                                  size_t workspace_bytes, dibr_b200_stream_t stream) {
  if (const int e = topo_dims(num_vertices, num_faces, face_size)) return e;
  const int64_t FS = num_faces * face_size;
  if (!corner_ptr || !adj_ptr || !status || !workspace) return DIBR_B200_EINVAL;
  if (FS > 0 && (!faces || !corners || !adj)) return DIBR_B200_EINVAL;
  if (num_vertices > 0 && (!degree || !weight)) return DIBR_B200_EINVAL;
  const dibr_layout::MeshTopologyLayout l = dibr_layout::mesh_topology_layout(num_vertices, num_faces, face_size);
  char* o = carve(workspace, workspace_bytes, l.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  Topo t;
  t.V = num_vertices; t.S = face_size; t.R = 2; t.F = (int)num_faces; t.faces = faces;
  t.corner_ptr = corner_ptr; t.corners = corners; t.adj_ptr = adj_ptr; t.adj = adj; t.degree = degree;
  t.weight = weight; t.status = status;
  return topo_build(t, o, l.topo, (cudaStream_t)stream);
}

int dibr_b200_laplacian_apply(int batch, int num_vertices, int channels, const int32_t* adj_ptr, const int32_t* adj,
                              const float* weight, const float* x, int transpose, int smooth, float* y,
                              dibr_b200_stream_t stream) {
  if (batch < 0 || num_vertices < 0 || channels < 0) return DIBR_B200_EINVAL;
  const int64_t rows = (int64_t)batch * num_vertices;
  if (rows == 0 || channels == 0) return 0;
  if (!adj_ptr || !adj || !weight || !x || !y) return DIBR_B200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const int V = num_vertices;
#define DIBR_B200_APPLY(T, S, NAME3, NAME)                                                                   \
  if (channels == 3) {                                                                                       \
    Span s(NAME3, st);                                                                                       \
    laplacian_apply3_kernel<T, S><<<grid_for(rows, kThreads), kThreads, 0, st>>>(rows, V, adj_ptr, adj, weight, x, y); \
  } else {                                                                                                   \
    Span s(NAME, st);                                                                                        \
    const int64_t total = rows * channels;                                                                   \
    laplacian_apply_kernel<T, S><<<grid_for(total, kThreads), kThreads, 0, st>>>(total, V, channels, adj_ptr, adj, \
                                                                                 weight, x, y);              \
  }
  if (transpose) {
    if (smooth) { DIBR_B200_APPLY(true, true, "laplacian_apply3_kernel<T,smooth>", "laplacian_apply_kernel<T,smooth>") }
    else { DIBR_B200_APPLY(true, false, "laplacian_apply3_kernel<T>", "laplacian_apply_kernel<T>") }
  } else {
    if (smooth) { DIBR_B200_APPLY(false, true, "laplacian_apply3_kernel<smooth>", "laplacian_apply_kernel<smooth>") }
    else { DIBR_B200_APPLY(false, false, "laplacian_apply3_kernel", "laplacian_apply_kernel") }
  }
#undef DIBR_B200_APPLY
  return (int)cudaGetLastError();
}

int dibr_b200_vertex_average_forward(int batch, int num_vertices, int64_t num_faces, int face_size, int channels,
                                     const int32_t* corner_ptr, const int32_t* corners, const float* face_features,
                                     float* out, dibr_b200_stream_t stream) {
  if (batch < 0 || channels < 0) return DIBR_B200_EINVAL;
  if (const int e = topo_dims(num_vertices, num_faces, face_size)) return e;
  const int64_t total = (int64_t)batch * num_vertices * channels;
  if (total == 0) return 0;
  if (!corner_ptr || !out || (num_faces > 0 && (!corners || !face_features))) return DIBR_B200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  Span s("vertex_average_kernel", st);
  vertex_average_kernel<<<grid_for(total, kThreads), kThreads, 0, st>>>(total, num_vertices, num_faces * face_size,
                                                                        channels, corner_ptr, corners, face_features, out);
  return (int)cudaGetLastError();
}

int dibr_b200_vertex_average_backward(int batch, int num_vertices, int64_t num_faces, int face_size, int channels,
                                      const int64_t* faces, const int32_t* corner_ptr, const float* grad_out,
                                      float* grad_face_features, dibr_b200_stream_t stream) {
  if (batch < 0 || channels < 0) return DIBR_B200_EINVAL;
  if (const int e = topo_dims(num_vertices, num_faces, face_size)) return e;
  const int64_t FS = num_faces * face_size;
  const int64_t total = (int64_t)batch * FS * channels;
  if (total == 0) return 0;
  if (!faces || !corner_ptr || !grad_out || !grad_face_features) return DIBR_B200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  Span s("vertex_average_bwd_kernel", st);
  vertex_average_bwd_kernel<<<grid_for(total, kThreads), kThreads, 0, st>>>(total, num_vertices, FS, channels, faces,
                                                                            corner_ptr, grad_out, grad_face_features);
  return (int)cudaGetLastError();
}

int dibr_b200_mesh_dense(int num_vertices, int laplacian, const int32_t* adj_ptr, const int32_t* adj,
                         const float* weight, float* out, dibr_b200_stream_t stream) {
  if (num_vertices < 0) return DIBR_B200_EINVAL;
  if (num_vertices == 0) return 0;
  if (!adj_ptr || !adj || !out || (laplacian && !weight)) return DIBR_B200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n = (int64_t)num_vertices * num_vertices;
  const int64_t cap = (int64_t)132 * 64;
  const unsigned grid = (unsigned)(grid_for(n, kThreads) < cap ? grid_for(n, kThreads) : cap);
  if (laplacian) {
    Span s("dense_kernel<laplacian>", st);
    dense_kernel<true><<<grid, kThreads, 0, st>>>(num_vertices, adj_ptr, adj, weight, out);
  } else {
    Span s("dense_kernel<adjacency>", st);
    dense_kernel<false><<<grid, kThreads, 0, st>>>(num_vertices, adj_ptr, adj, weight, out);
  }
  return (int)cudaGetLastError();
}

int dibr_b200_adjacency_coo(int num_vertices, int64_t num_edges, const int32_t* adj_ptr, const int32_t* adj,
                            int64_t* indices, dibr_b200_stream_t stream) {
  if (num_vertices < 0 || num_edges < 0) return DIBR_B200_EINVAL;
  if (num_edges == 0) return 0;
  if (!adj_ptr || !adj || !indices) return DIBR_B200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  Span s("adjacency_coo_kernel", st);
  adjacency_coo_kernel<<<grid_for(32 * (int64_t)num_vertices, kThreads), kThreads, 0, st>>>(num_vertices, num_edges,
                                                                                            adj_ptr, adj, indices);
  return (int)cudaGetLastError();
}

size_t dibr_b200_loop_subdivision_workspace_bytes(int num_vertices, int64_t num_faces) {
  if (topo_dims(num_vertices, num_faces, 3)) return 0;
  return dibr_layout::subdivision_layout(num_vertices).bytes;
}

int dibr_b200_loop_subdivision_build(int num_vertices, int64_t num_faces, const int64_t* faces,
                                     const int32_t* corner_ptr, const int32_t* corners, const int32_t* adj_ptr,
                                     const int32_t* adj, int32_t* edge_ptr, int32_t* adj_edge, int32_t* face_edge,
                                     int32_t* edges, int64_t* new_faces, int32_t* status, void* workspace,
                                     size_t workspace_bytes, dibr_b200_stream_t stream) {
  if (const int e = topo_dims(num_vertices, num_faces, 3)) return e;
  if (!corner_ptr || !adj_ptr || !edge_ptr || !status || !workspace) return DIBR_B200_EINVAL;
  if (num_faces > 0 && (!faces || !corners || !adj || !adj_edge || !face_edge || !edges || !new_faces))
    return DIBR_B200_EINVAL;
  const dibr_layout::SubdivisionLayout l = dibr_layout::subdivision_layout(num_vertices);
  char* o = carve(workspace, workspace_bytes, l.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  Subdiv s;
  s.V = num_vertices; s.F = (int)num_faces; s.faces = faces;
  s.corner_ptr = corner_ptr; s.corners = corners; s.adj_ptr = adj_ptr; s.adj = adj;
  s.count = piece<int>(o, l.count); s.edge_ptr = edge_ptr; s.adj_edge = adj_edge; s.face_edge = face_edge;
  s.edges = (int4*)edges; s.new_faces = new_faces;
  cudaStream_t st = (cudaStream_t)stream;
  const int V = num_vertices;
  if (V > 0) { Span sp("subdiv_count_kernel", st); subdiv_count_kernel<<<grid_for(V, kThreads), kThreads, 0, st>>>(s); }
  if (int e = exclusive_scan(s.count, V, piece<int>(o, l.sums), edge_ptr, st)) return e;
  if (num_faces > 0) {
    const int64_t capacity = 6 * num_faces;       // the adjacency holds at most 2 * F * 3 entries
    { Span sp("subdiv_edges_kernel", st); subdiv_edges_kernel<true><<<grid_for(capacity, kThreads), kThreads, 0, st>>>(s, capacity); }
    { Span sp("subdiv_faces_kernel", st); subdiv_faces_kernel<<<grid_for(num_faces, kThreads), kThreads, 0, st>>>(s); }
  }
  cudaMemcpyAsync(status, edge_ptr + V, sizeof(int32_t), cudaMemcpyDeviceToDevice, st);
  return (int)cudaGetLastError();
}

int dibr_b200_loop_subdivision_forward(int batch, int num_vertices, int num_edges, const int32_t* adj_ptr,
                                       const int32_t* adj, const int32_t* edges, const int64_t* faces,
                                       const float* vertices, const float* alpha, float* out, float* alpha_out,
                                       dibr_b200_stream_t stream) {
  if (batch < 0 || num_vertices < 0 || num_edges < 0 || (int64_t)num_vertices + num_edges >= INT32_MAX)
    return DIBR_B200_EINVAL;
  if (alpha_out && !alpha) return DIBR_B200_EINVAL;
  const int64_t total = (int64_t)batch * (num_vertices + num_edges);
  if (total == 0) return 0;
  if (!adj_ptr || !out || (num_vertices > 0 && !vertices)) return DIBR_B200_EINVAL;
  if (num_edges > 0 && (!adj || !edges || !faces)) return DIBR_B200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const int4* e4 = (const int4*)edges;
  if (alpha) {
    Span s("subdiv_forward_kernel<alpha>", st);
    subdiv_forward_kernel<true><<<grid_for(total, kThreads), kThreads, 0, st>>>(
        total, num_vertices, num_edges, adj_ptr, adj, e4, faces, vertices, alpha, out, alpha_out);
  } else {
    Span s("subdiv_forward_kernel", st);
    subdiv_forward_kernel<false><<<grid_for(total, kThreads), kThreads, 0, st>>>(
        total, num_vertices, num_edges, adj_ptr, adj, e4, faces, vertices, nullptr, out, nullptr);
  }
  return (int)cudaGetLastError();
}

int dibr_b200_loop_subdivision_backward(int batch, int num_vertices, int num_edges, const int32_t* corner_ptr,
                                        const int32_t* corners, const int32_t* adj_ptr, const int32_t* adj,
                                        const int32_t* adj_edge, const int32_t* face_edge, const int32_t* edges,
                                        const float* vertices, const float* alpha, const float* grad_out,
                                        const float* grad_alpha_out, float* grad_vertices, float* grad_alpha,
                                        dibr_b200_stream_t stream) {
  if (batch < 0 || num_vertices < 0 || num_edges < 0 || (int64_t)num_vertices + num_edges >= INT32_MAX)
    return DIBR_B200_EINVAL;
  if ((grad_alpha_out || grad_alpha) && !alpha) return DIBR_B200_EINVAL;
  if (grad_alpha && !vertices) return DIBR_B200_EINVAL;
  const int64_t total = (int64_t)batch * num_vertices;
  if (total == 0 || (!grad_vertices && !grad_alpha)) return 0;
  if (!corner_ptr || !adj_ptr || !grad_out) return DIBR_B200_EINVAL;
  if (num_edges > 0 && (!corners || !adj || !adj_edge || !face_edge || !edges)) return DIBR_B200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const int4* e4 = (const int4*)edges;
  if (alpha) {
    Span s("subdiv_backward_kernel<alpha>", st);
    subdiv_backward_kernel<true><<<grid_for(total, kThreads), kThreads, 0, st>>>(
        total, num_vertices, num_edges, corner_ptr, corners, adj_ptr, adj, adj_edge, face_edge, e4, vertices, alpha,
        grad_out, grad_alpha_out, grad_vertices, grad_alpha);
  } else {
    Span s("subdiv_backward_kernel", st);
    subdiv_backward_kernel<false><<<grid_for(total, kThreads), kThreads, 0, st>>>(
        total, num_vertices, num_edges, corner_ptr, corners, adj_ptr, adj, adj_edge, face_edge, e4, vertices, nullptr,
        grad_out, nullptr, grad_vertices, nullptr);
  }
  return (int)cudaGetLastError();
}

size_t dibr_b200_tet_topology_workspace_bytes(int num_vertices, int64_t num_tets) {
  if (topo_dims(num_vertices, num_tets, 4, 3)) return 0;
  return dibr_layout::tet_topology_layout(num_vertices, num_tets).bytes;
}

int dibr_b200_tet_topology_build(int num_vertices, int64_t num_tets, const int64_t* tets, int32_t* adj_ptr,
                                 int32_t* adj, int32_t* edges, int32_t* adj_edge, int32_t* tet_edge, int32_t* status,
                                 void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream) {
  if (const int e = topo_dims(num_vertices, num_tets, 4, 3)) return e;
  if (!adj_ptr || !status || !workspace) return DIBR_B200_EINVAL;
  if (num_tets > 0 && (!tets || !adj || !edges || !adj_edge || !tet_edge)) return DIBR_B200_EINVAL;
  const dibr_layout::TetTopologyLayout l = dibr_layout::tet_topology_layout(num_vertices, num_tets);
  char* o = carve(workspace, workspace_bytes, l.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int V = num_vertices;
  Topo t;
  t.V = V; t.S = 4; t.R = 3; t.F = (int)num_tets; t.faces = tets;
  t.corner_ptr = piece<int>(o, l.corner_ptr); t.corners = piece<int>(o, l.corners); t.adj_ptr = adj_ptr; t.adj = adj;
  t.degree = piece<int>(o, l.degree); t.weight = piece<float>(o, l.weight); t.status = piece<int>(o, l.status);
  if (int e = topo_build(t, o, l.topo, st)) return e;
  // the topology's count (all zero again) and scan partials serve the edge numbering
  Subdiv s;
  s.V = V; s.F = (int)num_tets; s.faces = tets;
  s.corner_ptr = t.corner_ptr; s.corners = t.corners; s.adj_ptr = adj_ptr; s.adj = adj;
  s.count = t.count; s.edge_ptr = piece<int>(o, l.edge_ptr); s.adj_edge = adj_edge; s.face_edge = tet_edge;
  s.edges = nullptr; s.new_faces = nullptr; s.pairs = (int2*)edges;
  if (V > 0) { Span sp("subdiv_count_kernel", st); subdiv_count_kernel<<<grid_for(V, kThreads), kThreads, 0, st>>>(s); }
  if (int e = exclusive_scan(s.count, V, t.sums, s.edge_ptr, st)) return e;
  if (num_tets > 0) {
    const int64_t capacity = 12 * num_tets;       // the adjacency holds at most 3 * T * 4 entries
    { Span sp("subdiv_edges_kernel<pairs>", st); subdiv_edges_kernel<false><<<grid_for(capacity, kThreads), kThreads, 0, st>>>(s, capacity); }
    { Span sp("tet_edges_kernel", st); tet_edges_kernel<<<grid_for(num_tets, kThreads), kThreads, 0, st>>>(s); }
  }
  cudaMemcpyAsync(status, s.edge_ptr + V, sizeof(int32_t), cudaMemcpyDeviceToDevice, st);
  cudaMemcpyAsync(status + 1, t.status + 1, sizeof(int32_t), cudaMemcpyDeviceToDevice, st);
  cudaMemcpyAsync(status + 2, t.status, sizeof(int32_t), cudaMemcpyDeviceToDevice, st);
  return (int)cudaGetLastError();
}

int dibr_b200_marching_tets_case_table(int32_t* pairs) {
  if (!pairs) return DIBR_B200_EINVAL;
  for (int c = 0; c < 16; ++c) {
    const int n = __builtin_popcount(c) == 2 ? 2 : (__builtin_popcount(c) & 1);
    for (int k = 0; k < 6; ++k) {
      int a = -1, b = -1;
      if (k < 3 * n) mt_pair_slot(kMtCasesHost[c], k, &a, &b);
      pairs[12 * c + 2 * k] = a;
      pairs[12 * c + 2 * k + 1] = b;
    }
  }
  return 0;
}

// B*(E + 2T) flags and their scan must be indexable by int.
static int mt_dims(int batch, int V, int E, int64_t T) {
  if (batch < 0 || V < 0 || E < 0 || T < 0) return DIBR_B200_EINVAL;
  if ((int64_t)batch * ((int64_t)E + 2 * T) >= INT32_MAX || T > INT32_MAX / 12) return DIBR_B200_ESIZE;
  return 0;
}

size_t dibr_b200_marching_tets_workspace_bytes(int batch, int num_edges, int64_t num_tets) {
  if (mt_dims(batch, 0, num_edges, num_tets)) return 0;
  return dibr_layout::marching_tets_layout(batch, num_edges, num_tets).bytes;
}

int dibr_b200_marching_tets_count(int batch, int num_vertices, int num_edges, int64_t num_tets, const int32_t* edges,
                                  const int64_t* tets, const float* sdf, int32_t* scan, int32_t* counts,
                                  void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream) {
  if (const int e = mt_dims(batch, num_vertices, num_edges, num_tets)) return e;
  if (!scan || !workspace) return DIBR_B200_EINVAL;
  if (batch > 0 && !counts) return DIBR_B200_EINVAL;
  if (num_edges > 0 && !edges) return DIBR_B200_EINVAL;
  if (num_tets > 0 && !tets) return DIBR_B200_EINVAL;
  if (batch > 0 && num_vertices > 0 && !sdf) return DIBR_B200_EINVAL;
  const dibr_layout::MarchingTetsLayout l = dibr_layout::marching_tets_layout(batch, num_edges, num_tets);
  char* o = carve(workspace, workspace_bytes, l.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  MTets m = {};
  m.B = batch; m.V = num_vertices; m.E = num_edges; m.T = (int)num_tets;
  m.edges = (const int2*)edges; m.tets = tets; m.sdf = sdf; m.flags = piece<int>(o, l.flags); m.scan = scan;
  const int64_t n = (int64_t)batch * (num_edges + 2 * num_tets);
  int* sums = piece<int>(o, l.sums);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t classify = (int64_t)batch * (num_edges + num_tets);
  if (classify > 0) { Span s("mt_classify_kernel", st); mt_classify_kernel<<<grid_for(classify, kThreads), kThreads, 0, st>>>(m); }
  if (int e = exclusive_scan(m.flags, (int)n, sums, scan, st)) return e;
  if (batch > 0) { Span s("mt_counts_kernel", st); mt_counts_kernel<<<grid_for(batch, kThreads), kThreads, 0, st>>>(m, counts); }
  return (int)cudaGetLastError();
}

int dibr_b200_marching_tets_emit(int batch, int num_vertices, int num_edges, int64_t num_tets, const int32_t* edges,
                                 const int64_t* tets, const int32_t* tet_edge, const float* vertices, const float* sdf,
                                 const int32_t* scan, int32_t* vid, float* out_vertices, int64_t* out_faces,
                                 int64_t* out_tet_idx, dibr_b200_stream_t stream) {
  if (const int e = mt_dims(batch, num_vertices, num_edges, num_tets)) return e;
  const int64_t BE = (int64_t)batch * num_edges, BT = (int64_t)batch * num_tets;
  if (BE + BT == 0) return 0;
  if (!scan || !sdf || !out_vertices || !out_faces) return DIBR_B200_EINVAL;
  if (BE > 0 && (!edges || !vid || !vertices)) return DIBR_B200_EINVAL;
  if (BT > 0 && (!tets || !tet_edge || !vid)) return DIBR_B200_EINVAL;
  MTets m = {};
  m.B = batch; m.V = num_vertices; m.E = num_edges; m.T = (int)num_tets;
  m.edges = (const int2*)edges; m.tets = tets; m.tet_edge = tet_edge; m.x = vertices; m.sdf = sdf; m.scan = scan;
  m.vid = vid; m.out_v = out_vertices; m.out_f = out_faces; m.out_tet = out_tet_idx;
  cudaStream_t st = (cudaStream_t)stream;
  if (BE > 0) { Span s("mt_vertices_kernel", st); mt_vertices_kernel<<<grid_for(BE, kThreads), kThreads, 0, st>>>(m); }
  if (BT > 0) { Span s("mt_faces_kernel", st); mt_faces_kernel<<<grid_for(BT, kThreads), kThreads, 0, st>>>(m); }
  return (int)cudaGetLastError();
}

int dibr_b200_marching_tets_backward(int batch, int num_vertices, int num_edges, const int32_t* adj_ptr,
                                     const int32_t* adj, const int32_t* adj_edge, const float* vertices,
                                     const float* sdf, const int32_t* vid, const float* grad_out,
                                     float* grad_vertices, float* grad_sdf, dibr_b200_stream_t stream) {
  if (batch < 0 || num_vertices < 0 || num_edges < 0) return DIBR_B200_EINVAL;
  const int64_t total = (int64_t)batch * num_vertices;
  if (total == 0 || (!grad_vertices && !grad_sdf)) return 0;
  if (!adj_ptr || !vertices || !sdf) return DIBR_B200_EINVAL;
  if (num_edges > 0 && (!adj || !adj_edge || !vid || !grad_out)) return DIBR_B200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  Span s("mt_backward_kernel", st);
  mt_backward_kernel<<<grid_for(total, kThreads), kThreads, 0, st>>>(total, num_vertices, num_edges, adj_ptr, adj,
                                                                     adj_edge, vertices, sdf, vid, grad_out,
                                                                     grad_vertices, grad_sdf);
  return (int)cudaGetLastError();
}

int dibr_b200_tet_subdivide_forward(int batch, int num_vertices, int num_edges, int64_t num_tets, int channels,
                                    const int32_t* edges, const int64_t* tets, const int32_t* tet_edge,
                                    const float* vertices, const float* features, float* out_vertices,
                                    float* out_features, int64_t* out_tets, dibr_b200_stream_t stream) {
  if (batch < 0 || num_vertices < 0 || num_edges < 0 || num_tets < 0 || channels < 0) return DIBR_B200_EINVAL;
  if ((int64_t)num_vertices + num_edges >= INT32_MAX || num_tets > INT32_MAX / 12) return DIBR_B200_ESIZE;
  if (channels > 0 && (!features || !out_features)) return DIBR_B200_EINVAL;
  const int64_t total = (int64_t)batch * (num_vertices + num_edges);
  if (total > 0 && (!vertices || !out_vertices || (num_edges > 0 && !edges))) return DIBR_B200_EINVAL;
  if (out_tets && num_tets > 0 && (!tets || !tet_edge)) return DIBR_B200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  if (total > 0) {
    Span s("tet_subdivide_forward_kernel", st);
    tet_subdivide_forward_kernel<<<grid_for(total, kThreads), kThreads, 0, st>>>(
        total, num_vertices, num_edges, channels, (const int2*)edges, vertices, features, out_vertices, out_features);
  }
  if (out_tets && num_tets > 0) {
    Span s("tet_children_kernel", st);
    tet_children_kernel<<<grid_for(num_tets, kThreads), kThreads, 0, st>>>(num_vertices, (int)num_tets, tets, tet_edge,
                                                                           out_tets);
  }
  return (int)cudaGetLastError();
}

int dibr_b200_tet_subdivide_backward(int batch, int num_vertices, int num_edges, int channels, const int32_t* adj_ptr,
                                     const int32_t* adj, const int32_t* adj_edge, const float* grad_out_vertices,
                                     const float* grad_out_features, float* grad_vertices, float* grad_features,
                                     dibr_b200_stream_t stream) {
  if (batch < 0 || num_vertices < 0 || num_edges < 0 || channels < 0) return DIBR_B200_EINVAL;
  if ((int64_t)num_vertices + num_edges >= INT32_MAX) return DIBR_B200_ESIZE;
  if (grad_features && channels > 0 && !grad_out_features) return DIBR_B200_EINVAL;
  if (grad_vertices && !grad_out_vertices) return DIBR_B200_EINVAL;
  const int64_t total = (int64_t)batch * num_vertices;
  if (channels == 0) grad_features = nullptr;
  if (total == 0 || (!grad_vertices && !grad_features)) return 0;
  if (!adj_ptr || (num_edges > 0 && (!adj || !adj_edge))) return DIBR_B200_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  Span s("tet_subdivide_backward_kernel", st);
  tet_subdivide_backward_kernel<<<grid_for(total, kThreads), kThreads, 0, st>>>(
      total, num_vertices, num_edges, channels, adj_ptr, adj, adj_edge, grad_out_vertices, grad_out_features,
      grad_vertices, grad_features);
  return (int)cudaGetLastError();
}

}  // extern "C"
