// scan.cuh — the device-wide exclusive scan of csrc/mesh_topology.cu, shared with the other sources
// that size their outputs from per-element counts (csrc/marching_cubes.cu).
#pragma once
#include <cuda_runtime.h>

namespace dibr_b200_detail {

constexpr int kScanTile = 4096;   // elements per CTA: `sums` holds ceil(n / kScanTile) ints

// Exclusive scan in[n] -> out[n + 1] (out[n] = the total), enqueued on st; `in` and `out` must not
// overlap.  Returns a cudaError_t.
int exclusive_scan(const int* in, int n, int* sums, int* out, cudaStream_t st);

}  // namespace dibr_b200_detail
