// row_sort.cuh — ascending in-place sorts of one CSR row of ints, shared by the sources that make a
// CSR deterministic after an atomic-cursor fill (csrc/mesh_topology.cu, csrc/point_mesh_distance.cu):
// one thread sorts a short row, one CTA sorts a long one.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

// One thread: insertion sort of a[0, n).
__device__ __forceinline__ void insertion_sort(int* a, int n) {
  for (int i = 1; i < n; ++i) {
    const int x = a[i];
    int j = i - 1;
    while (j >= 0 && a[j] > x) { a[j + 1] = a[j]; --j; }
    a[j + 1] = x;
  }
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

}  // namespace
