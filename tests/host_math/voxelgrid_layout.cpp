// TEST-ONLY: compiles the voxel-grid fill layout of kaolin_b200/csrc/op_layouts.h as plain C++ (g++) so
// that tests/test_voxelgrid_ops_cpu.py can check where its piece lies, for any workspace pointer, on a
// CPU-only box.
#include <cstdint>
#include <cstddef>
#include "../../kaolin_b200/csrc/op_layouts.h"

using namespace dibr_layout;

extern "C" {

// out = {total, labels.at, labels.bytes}.
void vg_layout(int64_t batch, int64_t voxels, int64_t* out) {
  const VoxelgridFillLayout L = voxelgrid_fill_layout(batch, voxels);
  out[0] = (int64_t)L.bytes;
  out[1] = (int64_t)L.labels.at;
  out[2] = (int64_t)L.labels.bytes;
}

// The offset of the origin from a workspace at `ws` of `ws_bytes`, or -1 when a layout of `bytes` does not fit.
int64_t vg_carve(uint64_t ws, uint64_t ws_bytes, uint64_t bytes) {
  char* o = carve((void*)(uintptr_t)ws, (size_t)ws_bytes, (size_t)bytes);
  return o ? (int64_t)((uintptr_t)o - (uintptr_t)ws) : -1;
}

}  // extern "C"
