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
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dibr_b200.h"

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

constexpr int kScanThreads = 1024;
constexpr int kScanTile = kScanThreads * 4;   // elements per CTA of the scan
constexpr int kShortRow = 32;                 // rows of at most this many corners are sorted by one thread
constexpr int kLongCtas = 132;                // CTAs that share out the long rows
constexpr int kThreads = 256;

__host__ __device__ inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

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

int exclusive_scan(const int* in, int n, int* sums, int* out, cudaStream_t st) {
  if (n == 0) return (int)cudaMemsetAsync(out, 0, sizeof(int), st);
  const int tiles = (int)((n + kScanTile - 1) / kScanTile);
  { Span s("scan_reduce_kernel", st); scan_reduce_kernel<<<tiles, kScanThreads, 0, st>>>(in, n, sums); }
  { Span s("scan_tiles_kernel", st); scan_tiles_kernel<<<1, kScanThreads, 0, st>>>(sums, tiles); }
  { Span s("scan_apply_kernel", st); scan_apply_kernel<<<tiles, kScanThreads, 0, st>>>(in, n, sums, out); }
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Build.
struct Topo {
  int V, S;
  int F;              // fits: 2*F*S < 2^31 is checked on the host
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
// and its two raw neighbours; the row sort below puts them in order.  Corners with an index outside
// [0, V) were counted nowhere and write nothing.
__global__ void __launch_bounds__(kThreads) topo_fill_kernel(Topo t) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= (int64_t)t.F * t.S) return;
  const int64_t v = t.faces[c];
  if (!valid_vertex(v, t.V)) return;
  const int f = (int)(c / t.S), k = (int)(c - (int64_t)f * t.S);
  const int p = t.corner_ptr[v] + atomicSub(t.count + v, 1) - 1;
  t.corners[p] = k * t.F + f;
  const int64_t* row = t.faces + (int64_t)f * t.S;
  t.raw[2 * (int64_t)p] = (int)row[k + 1 == t.S ? 0 : k + 1];
  t.raw[2 * (int64_t)p + 1] = (int)row[k == 0 ? t.S - 1 : k - 1];
}

__device__ __forceinline__ void insertion_sort(int* a, int n) {
  for (int i = 1; i < n; ++i) {
    const int x = a[i];
    int j = i - 1;
    while (j >= 0 && a[j] > x) { a[j + 1] = a[j]; --j; }
    a[j + 1] = x;
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
  int* nb = t.raw + 2 * (int64_t)b;
  insertion_sort(nb, 2 * n);
  int u = 0;
  for (int i = 0; i < 2 * n; ++i)
    if (i == 0 || nb[i] != nb[u - 1]) nb[u++] = nb[i];
  finish_row(t, v, u);
}

// Ascending bitonic network over a[0, n) in global memory, one CTA, any n: the "flip" form sorts
// every block of size k ascending, so a missing partner (index >= n) stands for +inf and is skipped.
__device__ void block_bitonic_sort(int* a, int64_t n) {
  int64_t n2 = 1;
  while (n2 < n) n2 <<= 1;
  for (int64_t k = 2; k <= n2; k <<= 1) {
    for (int64_t s = k >> 1; s > 0; s >>= 1) {
      for (int64_t p = threadIdx.x; p < (n2 >> 1); p += blockDim.x) {
        const int64_t blk = p / s, off = p - blk * s;
        const int64_t i = blk * 2 * s + off;
        const int64_t j = s == (k >> 1) ? blk * 2 * s + 2 * s - 1 - off : i + s;
        if (j < n) {
          const int x = a[i], y = a[j];
          if (x > y) { a[i] = y; a[j] = x; }
        }
      }
      __syncthreads();
    }
  }
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
    int* nb = t.raw + 2 * (int64_t)b;
    const int m = 2 * n;
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
  const int* src = t.raw + 2 * (int64_t)t.corner_ptr[v];
  const int b = t.adj_ptr[v], n = t.adj_ptr[v + 1] - b;
  for (int i = lane; i < n; i += 32) t.adj[b + i] = src[i];
}

struct TopoLayout {
  size_t count, raw, sums, long_rows, long_count, bytes;
};

TopoLayout topo_layout(int V, int64_t corners) {
  TopoLayout l;
  const size_t tiles = (size_t)(V + kScanTile - 1) / kScanTile + 1;
  l.count = 0;
  l.raw = align_up(l.count + sizeof(int) * (size_t)V, 256);
  l.sums = align_up(l.raw + sizeof(int) * 2 * (size_t)corners, 256);
  l.long_rows = align_up(l.sums + sizeof(int) * tiles, 256);
  l.long_count = align_up(l.long_rows + sizeof(int) * (size_t)V, 256);
  l.bytes = l.long_count + 256;
  return l;
}

// 0, or the error: V must leave room for V + 1 offsets, and the 2*F*S raw neighbour entries (so
// every offset and every key k*F + f) must fit a 32-bit int.
int topo_dims(int V, int64_t F, int S) {
  if (V < 0 || F < 0 || S < 3) return DIBR_B200_EINVAL;
  if (V == INT32_MAX || F > (int64_t)INT32_MAX / S / 2) return DIBR_B200_ESIZE;
  return 0;
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

}  // namespace

extern "C" {

size_t dibr_b200_mesh_topology_workspace_bytes(int num_vertices, int64_t num_faces, int face_size) {
  if (topo_dims(num_vertices, num_faces, face_size)) return 0;
  return topo_layout(num_vertices, num_faces * face_size).bytes;
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
  const TopoLayout l = topo_layout(num_vertices, FS);
  if (workspace_bytes < l.bytes) return DIBR_B200_EWORKSPACE;
  char* ws = (char*)workspace;
  Topo t;
  t.V = num_vertices; t.S = face_size; t.F = (int)num_faces; t.faces = faces;
  t.corner_ptr = corner_ptr; t.corners = corners; t.adj_ptr = adj_ptr; t.adj = adj; t.degree = degree;
  t.weight = weight; t.status = status;
  t.count = (int*)(ws + l.count); t.raw = (int*)(ws + l.raw); t.sums = (int*)(ws + l.sums);
  t.long_rows = (int*)(ws + l.long_rows); t.long_count = (int*)(ws + l.long_count);
  cudaStream_t st = (cudaStream_t)stream;
  const int V = num_vertices;
  if (cudaMemsetAsync(status, 0, 2 * sizeof(int), st) != cudaSuccess) return (int)cudaGetLastError();
  if (V > 0 && cudaMemsetAsync(t.count, 0, sizeof(int) * (size_t)V, st) != cudaSuccess) return (int)cudaGetLastError();
  if (cudaMemsetAsync(t.long_count, 0, sizeof(int), st) != cudaSuccess) return (int)cudaGetLastError();
  if (FS > 0) { Span s("topo_count_kernel", st); topo_count_kernel<<<grid_for(FS, kThreads), kThreads, 0, st>>>(t); }
  if (int e = exclusive_scan(t.count, V, t.sums, corner_ptr, st)) return e;
  if (FS > 0) { Span s("topo_fill_kernel", st); topo_fill_kernel<<<grid_for(FS, kThreads), kThreads, 0, st>>>(t); }
  if (V > 0) {
    { Span s("topo_sort_rows_kernel", st); topo_sort_rows_kernel<<<grid_for(V, kThreads), kThreads, 0, st>>>(t); }
    { Span s("topo_sort_long_kernel", st); topo_sort_long_kernel<<<kLongCtas, kScanThreads, 0, st>>>(t); }
  }
  if (int e = exclusive_scan(degree, V, t.sums, adj_ptr, st)) return e;
  {
    Span s("topo_compact_kernel", st);
    topo_compact_kernel<<<grid_for(32 * (int64_t)(V > 0 ? V : 1), kThreads), kThreads, 0, st>>>(t);
  }
  return (int)cudaGetLastError();
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

}  // extern "C"
