// grid_bins.cuh — the per-view uniform grid that DefTet (deftet.cu) and check_sign (check_sign.cu) bin
// their faces on.  A face is described by its 2-D box, float4 {lo0, lo1, hi0, hi1} at bbox[b * F + f];
// the grid of view b is G x G cells laid over bounds[b] = {lo0, lo1, G / width0, G / width1}.
//   count:  grid_bin_kernel<kClosed, false> adds every face to the counters of the cells its box
//           covers, or, when that is more than kMaxCells cells, to the view's wide-list counter;
//   scan:   grid_scan_kernel turns the counters into per-view offsets (one CTA per view) and zeroes them;
//   fill:   grid_bin_kernel<kClosed, true> repeats the count and stores the face ids.
// Within a cell the ids are in no particular order (atomics); both users only need the set.
// The cell of a coordinate, clamp((int)((v - lo) * inv), 0, G - 1), is monotone in v under
// round-to-nearest (a subtraction of a fixed lo, a product with a fixed inv >= 0, a clamp) and sends NaN
// to cell 0 and +-inf to the border cells, so a point whose coordinate lies in [box lo, box hi] always
// lands in a cell of the box's cell range.  kClosed picks the box test the face's user applies:
//   false  half-open [lo, hi) (DefTet): an empty or NaN box (!(hi > lo)) holds no point and is dropped;
//   true   closed [lo, hi] (check_sign): only a NaN box (!(hi >= lo)) is dropped.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "op_layouts.h"

namespace {

using dibr_layout::grid_side;     // the grid's side for F faces per view
using dibr_layout::kMaxCells;     // cells a face may be inserted in; wider faces -> the view's wide list
constexpr unsigned kGridFull = 0xffffffffu;

struct Grid {
  int B, F, P, G;
  const float* bounds;   // [B][4] lo0, lo1, G/width0, G/width1
  int* cnt;              // [B][G*G + 1] (last: wide list length)
  int* off;              // [B][G*G + 1]
  int* entries;          // [B][F*kMaxCells]
  int* wide;             // [B][F]
};

__device__ __forceinline__ int cell_of(float v, float lo, float inv, int G) {
  const float c = (v - lo) * inv;
  // NaN -> 0; the clamp keeps points on the upper border (and anything outside) in range
  return (int)fminf(fmaxf(c, 0.f), (float)(G - 1));
}

// cells whose points can pass the face's box test (conservative)
template <bool kClosed>
__device__ __forceinline__ bool face_cells(const Grid& g, int b, int64_t face, const float* bbox, int& cx0, int& cx1,
                                           int& cy0, int& cy1) {
  const float4 bb = __ldg(reinterpret_cast<const float4*>(bbox) + face);
  const float* bd = g.bounds + 4 * b;
  if (kClosed ? (!(bb.z >= bb.x) || !(bb.w >= bb.y)) : (!(bb.z > bb.x) || !(bb.w > bb.y))) return false;
  cx0 = cell_of(bb.x, bd[0], bd[2], g.G); cx1 = cell_of(bb.z, bd[0], bd[2], g.G);
  cy0 = cell_of(bb.y, bd[1], bd[3], g.G); cy1 = cell_of(bb.w, bd[1], bd[3], g.G);
  return true;
}

template <bool kClosed, bool FILL>
__global__ void __launch_bounds__(256) grid_bin_kernel(Grid g, const float* __restrict__ bbox) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)g.B * g.F) return;
  const int b = (int)(i / g.F), f = (int)(i - (int64_t)b * g.F);
  int cx0, cx1, cy0, cy1;
  if (!face_cells<kClosed>(g, b, i, bbox, cx0, cx1, cy0, cy1)) return;
  const int ncell = g.G * g.G;
  int* cnt = g.cnt + (size_t)b * (ncell + 1);
  if ((cx1 - cx0 + 1) * (cy1 - cy0 + 1) > kMaxCells) {
    const int pos = atomicAdd(cnt + ncell, 1);
    if (FILL) g.wide[(size_t)b * g.F + pos] = f;
    return;
  }
  for (int cy = cy0; cy <= cy1; ++cy)
    for (int cx = cx0; cx <= cx1; ++cx) {
      const int c = cy * g.G + cx;
      const int pos = atomicAdd(cnt + c, 1);
      if (FILL) g.entries[(size_t)b * g.F * kMaxCells + g.off[(size_t)b * (ncell + 1) + c] + pos] = f;
    }
}

// exclusive scan of the G*G cell counters of one view (the wide-list counter is only reset)
__global__ void __launch_bounds__(1024) grid_scan_kernel(Grid g) {
  __shared__ int warp_sums[32];
  __shared__ int carry;
  const int ncell = g.G * g.G;
  int* cnt = g.cnt + (size_t)blockIdx.x * (ncell + 1);
  int* off = g.off + (size_t)blockIdx.x * (ncell + 1);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) { carry = 0; off[ncell] = cnt[ncell]; cnt[ncell] = 0; }   // off[ncell] keeps the wide length
  __syncthreads();
  for (int base = 0; base < ncell; base += 1024) {
    const int i = base + tid;
    const int v = i < ncell ? cnt[i] : 0;
    int x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(kGridFull, x, d); if (lane >= d) x += y; }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int w = warp_sums[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(kGridFull, w, d); if (lane >= d) w += y; }
      warp_sums[lane] = w;
    }
    __syncthreads();
    const int excl = carry + (warp ? warp_sums[warp - 1] : 0) + x - v;
    if (i < ncell) { off[i] = excl; cnt[i] = 0; }
    __syncthreads();
    if (tid == 1023) carry = excl + v;
    __syncthreads();
  }
}

}  // namespace
