// scan.cuh — the device-wide exclusive scan of csrc/mesh_topology.cu, shared with the other sources
// that size their outputs from per-element counts (csrc/marching_cubes.cu).
#pragma once
#include <cuda_runtime.h>

#include "op_layouts.h"

namespace dibr_b200_detail {

using dibr_layout::kScanTile;   // elements per CTA

// Exclusive scan in[n] -> out[n + 1] (out[n] = the total), enqueued on st; `in` and `out` must not
// overlap, and `sums` holds dibr_layout::scan_sums_bytes(n).  Returns a cudaError_t.
int exclusive_scan(const int* in, int n, int* sums, int* out, cudaStream_t st);

}  // namespace dibr_b200_detail
