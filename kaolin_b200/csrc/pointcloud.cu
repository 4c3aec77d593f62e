// pointcloud.cu — kaolin.ops.pointcloud.farthest_point_sampling (the reference's kaolin/ops/pointcloud.py)
// for every view in one call, behind the C ABI of include/dibr_b200.h.  Points are (B, N, 3) float32,
// read in place through element strides.
//
// The contract fixes every output bit for any cluster size, path or run:
//   - d(p, q) = ((dx dx) + (dy dy)) + (dz dz), dx = p.x - q.x, each operation rounded to nearest
//     float32 with no contraction; a distance counts only when it is finite;
//   - the center c is the float32 rounding of S / n, S the float64 sum of the view's finite points
//     (all three coordinates finite) and n their count, (0, 0, 0) when n = 0.  S is summed in a fixed
//     order: chunks of kFpsChunk points in index order, each reduced by the tree i + h for
//     h = 512, 256, ..., 1 with a non-finite or missing point contributing 0, and the chunk sums
//     added in index order;
//   - round 0 keys every point by d(p, c); after the first point s0 the keys are reset to d(p, s0),
//     and after each later selection s_r, key(p) = min(key(p), d(p, s_r)); a distance that does not
//     count is skipped, so a point may have no key;
//   - each round takes the untaken point with the largest key, ties to the lowest index, or, if no
//     untaken point has a key, the lowest-index untaken point.
// A candidate is one 64-bit word, hi = 2 + the key's float bits (1 for an untaken point without a
// key, 0 for a taken one) and lo = ~index, so every maximum — over a thread's points, warp shuffles,
// shared memory, distributed shared memory or atomicMax — selects exactly that point, in any order.
// A key is held as a float: -1 for a taken point and +inf for none, so the min-update keeps both.
//
// Kernels:
//   - fps_chunk_sums_kernel: one CTA per (view, chunk) writes the chunk's float64 sums and count;
//   - fps_center_kernel: one thread per view adds its chunk sums in index order and divides;
//   - fps_kernel<false>, the cluster path: one thread-block cluster per view, its points split
//     across the CTAs and kept in registers (kFpsRegPoints per thread), then shared memory, for all k
//     rounds.  Each round min-updates the keys against the last winner, reduces to the 64-bit maximum
//     in the thread, the warp and the CTA, and pushes the CTA's candidate, with the point's
//     coordinates, into a double-buffered slot of every CTA of the cluster through distributed shared
//     memory; one cluster barrier ends the round, and every warp then reduces the slots itself.  A
//     round reads nothing from global memory;
//   - fps_kernel<true>, the grid path: one cooperative launch, a contiguous slice of a view per CTA,
//     its keys in registers, shared memory and, past those, the workspace.  Each round every CTA
//     adds its candidate to the view's slot with a 64-bit atomicMax, and one grid.sync() ends it.
//     Three rotating slots let the view's first CTA clear slot r + 1 during round r, two rounds after
//     its last read, without a second barrier.
// Round r's winner is kept by thread r mod kFpsThreads of every CTA and written out kFpsThreads
// rounds at a time.  Nothing spins on a flag besides the cluster barrier and the grid sync, and
// nothing is read back to the host.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/dibr_b200.h"
#include "op_layouts.h"

namespace cg = cooperative_groups;

// launch tracing (dibr_b200_trace_begin / _end), kept in dibr_b200.cu
namespace dibr_b200_detail {
bool span_open(const char* name, cudaStream_t st);
void span_close(cudaStream_t st);
}  // namespace dibr_b200_detail

namespace {

using dibr_layout::kFpsChunk;
using dibr_layout::kFpsRegPoints;
using dibr_layout::kFpsSmemPoints;
using dibr_layout::kFpsThreads;

struct Span {
  cudaStream_t st;
  bool on;
  Span(const char* name, cudaStream_t st_) : st(st_), on(dibr_b200_detail::span_open(name, st_)) {}
  ~Span() { if (on) dibr_b200_detail::span_close(st); }
};

constexpr int kWarps = kFpsThreads / 32;
constexpr int kMaxCluster = 16;
constexpr unsigned kFull = 0xffffffffu;
constexpr size_t kSmemMax = (size_t)kFpsThreads * kFpsSmemPoints * sizeof(float4);
constexpr int kChunkThreads = kFpsChunk / 2;   // two points per thread

int sm_count() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms > 0 ? sms : 132;
}

// ---------------------------------------------------------------------------------------------
// Center

struct View {
  const float* p;
  int64_t sb, sn, sc;
  __device__ __forceinline__ float3 at(int64_t b, int i) const {
    const float* q = p + b * sb + (int64_t)i * sn;
    return make_float3(q[0], q[sc], q[2 * sc]);
  }
};

// Point i of view b as float64 and its finite count, 0 when not finite or past the view.
__device__ __forceinline__ double4 finite_point(const View& v, int64_t b, int64_t i, int N) {
  if (i >= N) return make_double4(0.0, 0.0, 0.0, 0.0);
  const float3 p = v.at(b, (int)i);
  if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return make_double4(0.0, 0.0, 0.0, 0.0);
  return make_double4(p.x, p.y, p.z, 1.0);
}

__device__ __forceinline__ double4 add4(double4 a, double4 b) {
  return make_double4(__dadd_rn(a.x, b.x), __dadd_rn(a.y, b.y), __dadd_rn(a.z, b.z), __dadd_rn(a.w, b.w));
}

__device__ __forceinline__ double4 shfl_down4(double4 a, int h) {
  return make_double4(__shfl_down_sync(kFull, a.x, h), __shfl_down_sync(kFull, a.y, h),
                      __shfl_down_sync(kFull, a.z, h), __shfl_down_sync(kFull, a.w, h));
}

// s[i] = s[i] + s[i + h] for h = 512 (two points per thread), 256, 128, 64 in shared memory and 32 ... 1
// in warp 0's shuffles: the contract's tree.
__global__ void __launch_bounds__(kChunkThreads) fps_chunk_sums_kernel(View v, int N, int64_t pairs, int64_t chunks,
                                                                       double4* __restrict__ sums) {
  __shared__ double4 s[kChunkThreads];
  const int t = threadIdx.x;
  for (int64_t c = blockIdx.x; c < pairs; c += gridDim.x) {
    const int64_t b = c / chunks, i0 = (c - b * chunks) * kFpsChunk;
    s[t] = add4(finite_point(v, b, i0 + t, N), finite_point(v, b, i0 + t + kChunkThreads, N));
    __syncthreads();
    for (int h = kChunkThreads / 2; h >= 64; h >>= 1) {
      if (t < h) s[t] = add4(s[t], s[t + h]);
      __syncthreads();
    }
    if (t < 32) {
      double4 a = add4(s[t], s[t + 32]);
      for (int h = 16; h >= 1; h >>= 1) a = add4(a, shfl_down4(a, h));
      if (t == 0) sums[c] = a;
    }
    __syncthreads();
  }
}

__global__ void fps_center_kernel(int64_t B, int64_t chunks, const double4* __restrict__ sums,
                                  float4* __restrict__ centers) {
  for (int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
    const double4* s = sums + b * chunks;
    double4 S = s[0];
    for (int64_t c = 1; c < chunks; ++c) S = add4(S, s[c]);
    float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
    if (S.w > 0.0)
      out = make_float4(__double2float_rn(__ddiv_rn(S.x, S.w)), __double2float_rn(__ddiv_rn(S.y, S.w)),
                        __double2float_rn(__ddiv_rn(S.z, S.w)), 0.f);
    centers[b] = out;
  }
}

// ---------------------------------------------------------------------------------------------
// Rounds

struct Best {
  unsigned long long key;
  float x, y, z;
};

__device__ __forceinline__ float fps_dist(float px, float py, float pz, float qx, float qy, float qz) {
  const float dx = __fsub_rn(px, qx), dy = __fsub_rn(py, qy), dz = __fsub_rn(pz, qz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ unsigned long long fps_pack(float key, int idx) {
  const unsigned hi = key < 0.f ? 0u : key == INFINITY ? 1u : 2u + __float_as_uint(key);
  return ((unsigned long long)hi << 32) | (unsigned)~idx;
}

// One point's step of a round against q: round 0 (first) returns d(p, c) without storing it; later
// rounds min-update the stored key with d(p, w) and take w.  Returns the key the point competes with.
__device__ __forceinline__ float fps_step(float& key, float px, float py, float pz, int idx, bool first, float qx,
                                          float qy, float qz, int w) {
  const float d = fps_dist(px, py, pz, qx, qy, qz);
  const bool counts = d < INFINITY;   // false for inf and NaN
  if (first) return counts ? d : INFINITY;
  if (counts) key = fminf(key, d);
  if (idx == w) key = -1.f;
  return key;
}

__device__ __forceinline__ void offer(Best& b, unsigned long long key, float x, float y, float z) {
  if (key > b.key) {
    b.key = key;
    b.x = x;
    b.y = y;
    b.z = z;
  }
}

// The warp's largest candidate, in every lane.
__device__ __forceinline__ Best warp_max(Best b) {
  unsigned long long m = b.key;
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(kFull, m, o);
    m = other > m ? other : m;
  }
  const int src = __ffs(__ballot_sync(kFull, b.key == m)) - 1;
  return Best{m, __shfl_sync(kFull, b.x, src), __shfl_sync(kFull, b.y, src), __shfl_sync(kFull, b.z, src)};
}

struct FpsArgs {
  View v;
  int N, k;
  int per_view;      // CTAs per view: the cluster size, or the grid path's slices
  int64_t view0;     // the grid path's first view of this launch
  int n_cta;         // points per CTA (the last CTAs of a view may hold fewer, or none)
  int q;             // shared-memory points per thread
  const float4* centers;
  unsigned long long* slots;   // grid path: [B][3]
  float4* ws_points;           // grid path: [B][N]
  int64_t* out;
};

template <bool kGrid>
__global__ void __launch_bounds__(kFpsThreads, 1) fps_kernel(FpsArgs a) {
  extern __shared__ float4 sm_points[];
  __shared__ Best warp_best[kWarps];
  __shared__ Best cluster_best[2][kMaxCluster];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int part = (int)(blockIdx.x % a.per_view);
  const int64_t b = a.view0 + blockIdx.x / a.per_view;
  const int lo = (int)min((int64_t)part * a.n_cta, (int64_t)a.N);
  const int n = min(a.n_cta, a.N - lo);
  constexpr int R = kFpsRegPoints, T = kFpsThreads;
  const int reg_end = min(n, R * T), smem_end = min(n, (R + a.q) * T);

  float px[R], py[R], pz[R], pk[R];
#pragma unroll
  for (int i = 0; i < R; ++i) {
    const int j = t + T * i;
    float3 p = make_float3(0.f, 0.f, 0.f);
    if (j < reg_end) p = a.v.at(b, lo + j);
    px[i] = p.x;
    py[i] = p.y;
    pz[i] = p.z;
    pk[i] = INFINITY;
  }
  for (int j = R * T + t; j < smem_end; j += T) {
    const float3 p = a.v.at(b, lo + j);
    sm_points[j - R * T] = make_float4(p.x, p.y, p.z, INFINITY);
  }
  float4* ws = nullptr;
  if constexpr (kGrid) {
    ws = a.ws_points + b * a.N + lo;
    for (int j = smem_end + t; j < n; j += T) {
      const float3 p = a.v.at(b, lo + j);
      ws[j] = make_float4(p.x, p.y, p.z, INFINITY);
    }
  } else {
    cg::this_cluster().sync();   // every CTA of the cluster runs before any writes to its shared memory
  }

  const float4 c = a.centers[b];
  float qx = c.x, qy = c.y, qz = c.z;
  int w = -1, mine = 0;
  for (int r = 0; r < a.k; ++r) {
    const bool first = r == 0;
    Best best = {0ull, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const int j = t + T * i;
      if (j < reg_end) {
        const float key = fps_step(pk[i], px[i], py[i], pz[i], lo + j, first, qx, qy, qz, w);
        offer(best, fps_pack(key, lo + j), px[i], py[i], pz[i]);
      }
    }
    for (int j = R * T + t; j < smem_end; j += T) {
      float4 p = sm_points[j - R * T];
      const float key = fps_step(p.w, p.x, p.y, p.z, lo + j, first, qx, qy, qz, w);
      if (!first) sm_points[j - R * T].w = p.w;
      offer(best, fps_pack(key, lo + j), p.x, p.y, p.z);
    }
    if constexpr (kGrid) {
      for (int j = smem_end + t; j < n; j += T) {
        float4 p = ws[j];
        const float key = fps_step(p.w, p.x, p.y, p.z, lo + j, first, qx, qy, qz, w);
        if (!first) ws[j].w = p.w;
        offer(best, fps_pack(key, lo + j), p.x, p.y, p.z);
      }
    }
    best = warp_max(best);
    if (lane == 0) warp_best[warp] = best;
    __syncthreads();

    Best win;
    if constexpr (kGrid) {
      unsigned long long* slot = a.slots + 3 * b;
      if (warp == 0) {
        const Best cta = warp_max(lane < kWarps ? warp_best[lane] : Best{0ull, 0.f, 0.f, 0.f});
        if (lane == 0 && cta.key) atomicMax(slot + r % 3, cta.key);
        if (lane == 0 && part == 0) slot[(r + 1) % 3] = 0ull;
      }
      cg::this_grid().sync();
      const unsigned long long key = __ldcg(slot + r % 3);
      const float3 p = a.v.at(b, (int)~(unsigned)key);
      win = Best{key, p.x, p.y, p.z};
    } else {
      cg::cluster_group cluster = cg::this_cluster();
      const int buf = r & 1;
      if (warp == 0) {
        const Best cta = warp_max(lane < kWarps ? warp_best[lane] : Best{0ull, 0.f, 0.f, 0.f});
        if (lane < a.per_view) *cluster.map_shared_rank(&cluster_best[buf][part], lane) = cta;
      }
      cluster.sync();
      win = warp_max(lane < a.per_view ? cluster_best[buf][lane] : Best{0ull, 0.f, 0.f, 0.f});
    }
    w = (int)~(unsigned)win.key;
    qx = win.x;
    qy = win.y;
    qz = win.z;
    const int slot_r = r & (T - 1);
    if (slot_r == t) mine = w;
    if (part == 0 && (slot_r == T - 1 || r == a.k - 1) && t <= slot_r)
      a.out[b * a.k + (r - slot_r) + t] = mine;
  }
}

// ---------------------------------------------------------------------------------------------
// Host side.

int fps_shape(int64_t B, int64_t N, int64_t k) {
  if (B < 0 || N < 0 || k < 0) return DIBR_B200_EINVAL;
  if (N >= INT32_MAX) return DIBR_B200_ESIZE;
  if (k > N) return DIBR_B200_EINVAL;
  if (N > 0 && B > (INT64_MAX / 64) / N) return DIBR_B200_ESIZE;
  return 0;
}

// The largest cluster the current device launches with every CTA's shared-memory points in use.
int fps_max_cluster(int* out) {
  static int cached[64] = {0};
  int dev = 0;
  if (const cudaError_t e = cudaGetDevice(&dev)) return (int)e;
  if (dev >= 0 && dev < 64 && cached[dev]) {
    *out = cached[dev];
    return 0;
  }
  const void* fn = (const void*)fps_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  if (!e) e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemMax);
  if (e) return (int)e;
  int best = 0;
  for (int C = kMaxCluster; C >= 1 && !best; C >>= 1) {
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = C;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3(C);
    cfg.blockDim = dim3(kFpsThreads);
    cfg.dynamicSmemBytes = kSmemMax;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    int active = 0;
    if (cudaOccupancyMaxActiveClusters(&active, fn, &cfg) == cudaSuccess && active > 0) best = C;
    cudaGetLastError();   // a refused size is not an error of this call
  }
  if (!best) return (int)cudaErrorInvalidClusterSize;
  if (dev >= 0 && dev < 64) cached[dev] = best;
  *out = best;
  return 0;
}

int fps_cluster(const FpsArgs& base, int64_t B, const dibr_layout::FpsPlan& plan, cudaStream_t st) {
  FpsArgs a = base;
  a.per_view = plan.cluster;
  a.n_cta = (int)((a.N + plan.cluster - 1) / plan.cluster);
  a.q = plan.smem_points;
  if (B * plan.cluster > INT32_MAX) return DIBR_B200_ESIZE;
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = plan.cluster;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.gridDim = dim3((unsigned)(B * plan.cluster));
  cfg.blockDim = dim3(kFpsThreads);
  cfg.dynamicSmemBytes = (size_t)a.q * kFpsThreads * sizeof(float4);
  cfg.stream = st;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  int active = 0;
  if (const cudaError_t e = cudaOccupancyMaxActiveClusters(&active, (const void*)fps_kernel<false>, &cfg)) return (int)e;
  if (active < 1) return (int)cudaErrorInvalidClusterSize;
  Span sp("fps_kernel<cluster>", st);
  return (int)cudaLaunchKernelEx(&cfg, fps_kernel<false>, a);
}

int fps_grid(const FpsArgs& base, int64_t B, cudaStream_t st) {
  const void* fn = (const void*)fps_kernel<true>;
  if (const cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemMax))
    return (int)e;
  int per_sm = 0;
  if (const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kFpsThreads, kSmemMax))
    return (int)e;
  const int64_t ctas = (int64_t)per_sm * sm_count();
  if (ctas < 1) return (int)cudaErrorCooperativeLaunchTooLarge;
  if (const cudaError_t e = cudaMemsetAsync(base.slots, 0, (size_t)B * 3 * sizeof(unsigned long long), st)) return (int)e;
  Span sp("fps_kernel<grid>", st);
  for (int64_t v0 = 0; v0 < B; v0 += ctas) {
    const int64_t views = B - v0 < ctas ? B - v0 : ctas;
    FpsArgs a = base;
    a.view0 = v0;
    a.per_view = (int)(ctas / views);
    a.n_cta = (int)((a.N + a.per_view - 1) / a.per_view);
    a.q = dibr_layout::fps_smem_points(a.n_cta);
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeCooperative;
    at[0].val.cooperative = 1;
    cfg.gridDim = dim3((unsigned)(views * a.per_view));
    cfg.blockDim = dim3(kFpsThreads);
    cfg.dynamicSmemBytes = (size_t)a.q * kFpsThreads * sizeof(float4);
    cfg.stream = st;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    if (const cudaError_t e = cudaLaunchKernelEx(&cfg, fps_kernel<true>, a)) return (int)e;
  }
  return 0;
}

}  // namespace

int dibr_b200_farthest_point_sampling_workspace_bytes(int64_t batch, int64_t num_points, int64_t k,
                                                      size_t* workspace_bytes, int* path, int* cluster) {
  if (!workspace_bytes || !path || !cluster) return DIBR_B200_EINVAL;
  if (const int e = fps_shape(batch, num_points, k)) return e;
  int max_cluster = 0;
  if (batch * k > 0)
    if (const int e = fps_max_cluster(&max_cluster)) return e;
  const dibr_layout::FpsLayout L = dibr_layout::fps_layout(batch, num_points, k, max_cluster);
  *workspace_bytes = L.bytes;
  *path = L.plan.path;
  *cluster = L.plan.cluster;
  return 0;
}

int dibr_b200_farthest_point_sampling(int64_t batch, int64_t num_points, int64_t k, const float* points,
                                      int64_t stride_b, int64_t stride_n, int64_t stride_c, int64_t* out,
                                      void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream) {
  if (const int e = fps_shape(batch, num_points, k)) return e;
  if (batch * k == 0) return 0;
  if (!points || !out) return DIBR_B200_EINVAL;
  int max_cluster = 0;
  if (const int e = fps_max_cluster(&max_cluster)) return e;
  const dibr_layout::FpsLayout L = dibr_layout::fps_layout(batch, num_points, k, max_cluster);
  char* o = dibr_layout::carve(workspace, workspace_bytes, L.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const View v{points, stride_b, stride_n, stride_c};
  const int N = (int)num_points;
  const int64_t chunks = dibr_layout::fps_chunks(N), pairs = batch * chunks;
  double4* sums = dibr_layout::piece<double4>(o, L.chunk_sums);
  float4* centers = dibr_layout::piece<float4>(o, L.centers);
  {
    Span sp("fps_chunk_sums_kernel", st);
    const int64_t cap = 8LL * sm_count();
    fps_chunk_sums_kernel<<<(unsigned)(pairs < cap ? pairs : cap), kChunkThreads, 0, st>>>(v, N, pairs, chunks, sums);
  }
  {
    Span sp("fps_center_kernel", st);
    const int64_t blocks = (batch + 127) / 128;
    fps_center_kernel<<<(unsigned)(blocks < 1024 ? blocks : 1024), 128, 0, st>>>(batch, chunks, sums, centers);
  }
  if (const cudaError_t e = cudaGetLastError()) return (int)e;
  FpsArgs a = {};
  a.v = v;
  a.N = N;
  a.k = (int)k;
  a.centers = centers;
  a.slots = dibr_layout::piece<unsigned long long>(o, L.slots);
  a.ws_points = dibr_layout::piece<float4>(o, L.points);
  a.out = out;
  return L.plan.path == dibr_layout::kFpsCluster ? fps_cluster(a, batch, L.plan, st) : fps_grid(a, batch, st);
}
