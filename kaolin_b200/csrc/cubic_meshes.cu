// cubic_meshes.cu — kaolin.ops.conversions.voxelgrids_to_cubic_meshes ("Cubify", Mesh R-CNN) for every
// view in one launch per kernel, behind the C ABI of include/dibr_b200.h.
//
// Contract.  A view's grid (X, Y, Z) is read as float32 and padded with zeros; its corner lattice is
// (X+1) x (Y+1) x (Z+1) points p, numbered l = (p0 (Y+1) + p1) (Z+1) + p2.  Voxel p is named by its
// minimum corner.  Face (a, p) separates voxel p from voxel p - e_a and exists when
// d = rint(v(p) - v(p - e_a)) != 0 (float32 subtraction, round half to even, NaN != 0).  A voxel
// outside the grid reads 0, so a face exists only where p_b < dim_b and p_c < dim_c, b = (a+1) mod 3,
// c = (a+2) mod 3.  Its corners are c0 = p, c1 = p + e_b, c2 = p + e_c, c3 = p + e_b + e_c; its quad is
// [c0, c1, c3, c2], reversed when d < 0.  A view's faces come axis by axis, each axis in lattice
// order; as triangles, every quad's [q0, q3, q1] and then every quad's [q2, q1, q3].  The vertices
// are the lattice points some face uses, in lattice order, as float32 (p0, p1, p2).
//
// Passes (all views at once):
//   count  one thread per (view, lattice point), a view's lattice padded to whole 32-point words so
//          that a warp never spans two views.  The thread reads the 2x2x2 voxel block below its
//          point: the faces it owns are its block's three pairs along the axes through voxel p, and
//          the point is a used corner exactly when one of the block's 12 axis-aligned pairs has d != 0.
//          Ballots turn each flag into a word: faces x, y, z, corner, and the reversal of each face.
//          The popcounts of the face and corner words are the scan's input, laid out
//          [every view's face words: view, then axis, then word][every view's corner words], so
//          one exclusive scan gives every face its output row over all views and every corner its
//          vertex row.
//   totals per-view face and vertex counts, the one value the caller reads back.
//   emit   one thread per (view, lattice point) again, reading only the bit planes and the scan: a
//          rank is the scan at the word plus the popcount of the word's lower lanes.
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
constexpr int kPlanes = 7;   // faces x, y, z, corners, reversed x, y, z

struct Cm {
  int B, X, Y, Z;
  int LY, LZ;            // lattice sides Y + 1, Z + 1
  int L;                 // lattice points per view
  int W;                 // words per view and plane
  int BW;                // B W
  int n;                 // threads: B W 32, at most 4 B L (cm_setup)
  int64_t sb, sx, sy, sz;
  const void* grid;
  uint32_t* bits;        // [kPlanes][B W]: face words at (v 3 + a) W + w, corners at 3 B W + v W + w,
                         // reversals at 4 B W + (v 3 + a) W + w
  int* counts;           // [4 B W] popcounts of the face and corner words, indexed as the bits
  const int* scan;       // [4 B W + 1]
  int* sums;             // the scan's tile sums
};

// The voxel (i, j, k) of view v, 0 outside the grid.
template <typename T>
__device__ __forceinline__ float voxel(const Cm& m, const T* base, int i, int j, int k) {
  if ((unsigned)i >= (unsigned)m.X || (unsigned)j >= (unsigned)m.Y || (unsigned)k >= (unsigned)m.Z) return 0.f;
  return (float)__ldg(base + i * m.sx + j * m.sy + k * m.sz);
}

__device__ __forceinline__ bool face(float hi, float lo) { return !(rintf(__fsub_rn(hi, lo)) == 0.f); }
__device__ __forceinline__ bool reversed(float hi, float lo) { return rintf(__fsub_rn(hi, lo)) < 0.f; }

__device__ __forceinline__ void lattice_point(const Cm& m, int l, int* a, int* b, int* c) {
  *c = l % m.LZ;
  const int r = l / m.LZ;
  *b = r % m.LY;
  *a = r / m.LY;
}

// n is a multiple of 32 and so is the grid's stride, so every warp runs whole.  The loop index is 64-bit:
// n may come within one stride of 2^31 - 1, and t + stride must not wrap.
template <typename T>
__global__ void __launch_bounds__(kThreads) cm_count_kernel(Cm m) {
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m.n; t += stride) {
    const int v = (int)(t / (32 * m.W)), l = (int)(t - (int64_t)v * 32 * m.W);
    unsigned flags = 0;   // bits 0-2 faces, 3 corner, 4-6 reversals
    if (l < m.L) {
      int a, b, c;
      lattice_point(m, l, &a, &b, &c);
      const T* base = (const T*)m.grid + v * m.sb;
      float f[2][2][2];   // f[i][j][k] = voxel (a - i, b - j, c - k)
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int k = 0; k < 2; ++k) f[i][j][k] = voxel<T>(m, base, a - i, b - j, c - k);
      flags = face(f[0][0][0], f[1][0][0]) | face(f[0][0][0], f[0][1][0]) << 1 | face(f[0][0][0], f[0][0][1]) << 2 |
              reversed(f[0][0][0], f[1][0][0]) << 4 | reversed(f[0][0][0], f[0][1][0]) << 5 |
              reversed(f[0][0][0], f[0][0][1]) << 6;
      bool used = false;
#pragma unroll
      for (int x = 0; x < 2; ++x)
#pragma unroll
        for (int y = 0; y < 2; ++y)
          used |= face(f[0][x][y], f[1][x][y]) | face(f[x][0][y], f[x][1][y]) | face(f[x][y][0], f[x][y][1]);
      flags |= used << 3;
    }
    uint32_t word[kPlanes];
#pragma unroll
    for (int k = 0; k < kPlanes; ++k) word[k] = __ballot_sync(0xffffffffu, (flags >> k) & 1);
    if (lane < kPlanes) {
      const int w = l >> 5;
      const int at = lane < 3 ? (v * 3 + lane) * m.W + w
                   : lane == 3 ? 3 * m.BW + v * m.W + w
                               : 4 * m.BW + (v * 3 + lane - 4) * m.W + w;
      uint32_t mine = word[0];
#pragma unroll
      for (int k = 1; k < kPlanes; ++k) mine = lane == k ? word[k] : mine;
      m.bits[at] = mine;
      if (lane < 4) m.counts[at] = __popc(mine);
    }
  }
}

__global__ void __launch_bounds__(kThreads) cm_totals_kernel(Cm m, int* __restrict__ totals) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= m.B) return;
  totals[2 * v] = m.scan[(v + 1) * 3 * m.W] - m.scan[v * 3 * m.W];
  totals[2 * v + 1] = m.scan[3 * m.BW + (v + 1) * m.W] - m.scan[3 * m.BW + v * m.W];
}

// The vertex id, within its view, of lattice point q of the view whose corner words start at `cw`.
__device__ __forceinline__ int64_t corner_id(const Cm& m, int cw, int q, int first) {
  const int w = cw + (q >> 5);
  return __ldg(m.scan + w) - first + __popc(__ldg(m.bits + w) & ((1u << (q & 31)) - 1u));
}

template <bool kTri>
__global__ void __launch_bounds__(kThreads) cm_emit_kernel(Cm m, float* __restrict__ out_v,
                                                           int64_t* __restrict__ out_f) {
  const int lane = threadIdx.x & 31;
  const unsigned below = (1u << lane) - 1u;
  const int step[3] = {m.LY * m.LZ, m.LZ, 1};
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m.n; t += stride) {
    const int v = (int)(t / (32 * m.W)), l = (int)(t - (int64_t)v * 32 * m.W), w = l >> 5;
    const int fw = v * 3 * m.W + w, cw = 3 * m.BW + v * m.W;
    const uint32_t fx = __ldg(m.bits + fw), fy = __ldg(m.bits + fw + m.W), fz = __ldg(m.bits + fw + 2 * m.W);
    const uint32_t cs = __ldg(m.bits + cw + w);
    if (!((fx | fy | fz | cs) >> lane & 1)) continue;
    int a, b, c;
    lattice_point(m, l, &a, &b, &c);
    const int first = __ldg(m.scan + cw);
    if (cs >> lane & 1) {
      const int64_t row = __ldg(m.scan + cw + w) - __ldg(m.scan + 3 * m.BW) + __popc(cs & below);
      out_v[3 * row] = (float)a;
      out_v[3 * row + 1] = (float)b;
      out_v[3 * row + 2] = (float)c;
    }
    const int view_face0 = __ldg(m.scan + v * 3 * m.W);
    const int view_faces = __ldg(m.scan + (v + 1) * 3 * m.W) - view_face0;
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) {
      const uint32_t word = ax == 0 ? fx : ax == 1 ? fy : fz;
      if (!(word >> lane & 1)) continue;
      const int at = fw + ax * m.W;
      const int64_t row = __ldg(m.scan + at) + __popc(word & below);
      const int sb = step[(ax + 1) % 3], sc = step[(ax + 2) % 3];
      const int64_t c0 = corner_id(m, cw, l, first), c1 = corner_id(m, cw, l + sb, first);
      const int64_t c2 = corner_id(m, cw, l + sc, first), c3 = corner_id(m, cw, l + sb + sc, first);
      int64_t q[4] = {c0, c1, c3, c2};
      if (__ldg(m.bits + 4 * m.BW + at) >> lane & 1) {
        q[0] = c2; q[1] = c3; q[2] = c1; q[3] = c0;
      }
      if (kTri) {
        int64_t* t0 = out_f + 3 * (2 * (int64_t)view_face0 + (row - view_face0));
        int64_t* t1 = t0 + 3 * (int64_t)view_faces;
        t0[0] = q[0]; t0[1] = q[3]; t0[2] = q[1];
        t1[0] = q[2]; t1[1] = q[1]; t1[2] = q[3];
      } else {
        int64_t* o = out_f + 4 * row;
        o[0] = q[0]; o[1] = q[1]; o[2] = q[2]; o[3] = q[3];
      }
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
  return (unsigned)(need < cap ? need : cap);
}

// Sizes and their index bounds: a view's lattice and 4 B L (the largest total the scan could reach,
// and a bound on its length and on the thread count n) must stay below 2^31 - 1.  The grid-stride
// loops step a 64-bit index, so n may come as close to that as it likes.
int cm_setup(Cm* m, int64_t batch, int64_t X, int64_t Y, int64_t Z) {
  if (batch < 0 || X < 1 || Y < 1 || Z < 1) return DIBR_B200_EINVAL;
  if (X >= INT32_MAX || Y >= INT32_MAX || Z >= INT32_MAX) return DIBR_B200_ESIZE;
  int64_t L = (X + 1) * (Y + 1);
  if (L >= INT32_MAX) return DIBR_B200_ESIZE;
  L *= Z + 1;
  if (L >= INT32_MAX) return DIBR_B200_ESIZE;
  if (batch >= INT32_MAX || batch * L > (INT32_MAX - 1) / 4) return DIBR_B200_ESIZE;
  if (m) {
    *m = Cm{};
    m->B = (int)batch; m->X = (int)X; m->Y = (int)Y; m->Z = (int)Z;
    m->LY = (int)Y + 1; m->LZ = (int)Z + 1; m->L = (int)L;
    m->W = (int)dibr_layout::cubic_meshes_words(L);
    m->BW = m->B * m->W;
    m->n = m->BW * 32;
  }
  return 0;
}

// The workspace's pieces in m, or an error.
int cm_carve(Cm* m, void* workspace, size_t workspace_bytes) {
  if (!workspace) return DIBR_B200_EINVAL;
  const dibr_layout::CubicMeshesLayout l = dibr_layout::cubic_meshes_layout(m->B, m->L);
  char* o = dibr_layout::carve(workspace, workspace_bytes, l.bytes);
  if (!o) return DIBR_B200_EWORKSPACE;
  m->bits = dibr_layout::piece<uint32_t>(o, l.bits);
  m->counts = dibr_layout::piece<int>(o, l.counts);
  m->scan = dibr_layout::piece<int>(o, l.scan);
  m->sums = dibr_layout::piece<int>(o, l.sums);
  return 0;
}

}  // namespace

int dibr_b200_cubic_meshes_workspace_bytes(int64_t batch, int64_t X, int64_t Y, int64_t Z, size_t* workspace_bytes) {
  if (!workspace_bytes) return DIBR_B200_EINVAL;
  Cm m;
  if (const int e = cm_setup(&m, batch, X, Y, Z)) return e;
  *workspace_bytes = dibr_layout::cubic_meshes_layout(m.B, m.L).bytes;
  return 0;
}

int dibr_b200_cubic_meshes_count(int64_t batch, int64_t X, int64_t Y, int64_t Z, int dtype, const void* grid,
                                 int64_t stride_b, int64_t stride_x, int64_t stride_y, int64_t stride_z,
                                 int32_t* totals, void* workspace, size_t workspace_bytes,
                                 dibr_b200_stream_t stream) {
  Cm m;
  if (const int e = cm_setup(&m, batch, X, Y, Z)) return e;
  if (dtype != DIBR_B200_DTYPE_F32 && dtype != DIBR_B200_DTYPE_U8) return DIBR_B200_EINVAL;
  if (batch > 0 && (!grid || !totals)) return DIBR_B200_EINVAL;
  if (const int e = cm_carve(&m, workspace, workspace_bytes)) return e;
  if (batch == 0) return 0;
  m.sb = stride_b; m.sx = stride_x; m.sy = stride_y; m.sz = stride_z;
  m.grid = grid;
  cudaStream_t st = (cudaStream_t)stream;
  {
    Span s("cm_count_kernel", st);
    if (dtype == DIBR_B200_DTYPE_F32)
      cm_count_kernel<float><<<grid_stride_ctas(m.n), kThreads, 0, st>>>(m);
    else
      cm_count_kernel<uint8_t><<<grid_stride_ctas(m.n), kThreads, 0, st>>>(m);
  }
  if (const int e = dibr_b200_detail::exclusive_scan(m.counts, 4 * m.BW, m.sums, (int*)m.scan, st)) return e;
  {
    Span s("cm_totals_kernel", st);
    cm_totals_kernel<<<(m.B + kThreads - 1) / kThreads, kThreads, 0, st>>>(m, totals);
  }
  return (int)cudaGetLastError();
}

int dibr_b200_cubic_meshes_emit(int64_t batch, int64_t X, int64_t Y, int64_t Z, int is_trimesh, float* out_vertices,
                                int64_t* out_faces, const void* workspace, size_t workspace_bytes,
                                dibr_b200_stream_t stream) {
  Cm m;
  if (const int e = cm_setup(&m, batch, X, Y, Z)) return e;
  if (batch > 0 && (!out_vertices || !out_faces)) return DIBR_B200_EINVAL;
  if (const int e = cm_carve(&m, (void*)workspace, workspace_bytes)) return e;
  if (batch == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  Span s("cm_emit_kernel", st);
  if (is_trimesh)
    cm_emit_kernel<true><<<grid_stride_ctas(m.n), kThreads, 0, st>>>(m, out_vertices, out_faces);
  else
    cm_emit_kernel<false><<<grid_stride_ctas(m.n), kThreads, 0, st>>>(m, out_vertices, out_faces);
  return (int)cudaGetLastError();
}
