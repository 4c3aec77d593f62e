// TEST-ONLY: compiles the farthest-point-sampling plan and layout of kaolin_b200/csrc/op_layouts.h as plain
// C++ (g++) so that tests/test_pointcloud_cpu.py can check the path, the cluster size and where each
// piece lies, for any workspace pointer, on a CPU-only box.
#include <cstdint>
#include <cstddef>
#include "../../kaolin_b200/csrc/op_layouts.h"

using namespace dibr_layout;

extern "C" {

// out = {path, cluster, smem_points, total, chunk_sums.at, .bytes, centers.at, .bytes, slots.at, .bytes,
//        points.at, .bytes}.
void fps_layout_of(int64_t B, int64_t N, int64_t k, int max_cluster, int64_t* out) {
  const FpsLayout L = fps_layout(B, N, k, max_cluster);
  const Piece pieces[4] = {L.chunk_sums, L.centers, L.slots, L.points};
  out[0] = L.plan.path;
  out[1] = L.plan.cluster;
  out[2] = L.plan.smem_points;
  out[3] = (int64_t)L.bytes;
  for (int i = 0; i < 4; ++i) {
    out[4 + 2 * i] = (int64_t)pieces[i].at;
    out[5 + 2 * i] = (int64_t)pieces[i].bytes;
  }
}

// {threads, register points, shared-memory points per thread, chunk}.
void fps_constants(int64_t* out) {
  out[0] = kFpsThreads;
  out[1] = kFpsRegPoints;
  out[2] = kFpsSmemPoints;
  out[3] = kFpsChunk;
}

// The offset of the origin from a workspace at `ws` of `ws_bytes`, or -1 when a layout of `bytes` does not fit.
int64_t fps_carve(uint64_t ws, uint64_t ws_bytes, uint64_t bytes) {
  char* o = carve((void*)(uintptr_t)ws, (size_t)ws_bytes, (size_t)bytes);
  return o ? (int64_t)((uintptr_t)o - (uintptr_t)ws) : -1;
}

}  // extern "C"
