// TEST-ONLY: compiles the surface-sampling layouts of kaolin_b200/csrc/op_layouts.h as plain C++ (g++)
// so that tests/test_sample_points_cpu.py can check where each piece lies, for any workspace pointer,
// on a CPU-only box.
#include <cstdint>
#include <cstddef>
#include <initializer_list>
#include "../../kaolin_b200/csrc/op_layouts.h"

using namespace dibr_layout;

extern "C" {

// out[0] = the total, then (at, bytes) of every piece: forward (cdf, coarse, tile_sum, tile_flag, carry,
// view_flag) when backward == 0, else (corner_grad, count, off, sums, ids, long_rows, long_count).
// Returns the number of values written.
int sp_layout(int backward, int B, int64_t nf, int N, int64_t tsize, int64_t* out) {
  int n = 1;
  if (!backward) {
    const SamplePointsForwardLayout L = sample_points_forward_layout(B, nf);
    out[0] = (int64_t)L.bytes;
    for (const Piece& p : {L.cdf, L.coarse, L.tile_sum, L.tile_flag, L.carry, L.view_flag}) {
      out[n] = (int64_t)p.at; out[n + 1] = (int64_t)p.bytes; n += 2;
    }
    return n;
  }
  const SamplePointsBackwardLayout L = sample_points_backward_layout(B, nf, N, (size_t)tsize);
  out[0] = (int64_t)L.bytes;
  for (const Piece& p : {L.corner_grad, L.count, L.off, L.sums, L.ids, L.long_rows, L.long_count}) {
    out[n] = (int64_t)p.at; out[n + 1] = (int64_t)p.bytes; n += 2;
  }
  return n;
}

// The offset of the origin from a workspace at `ws` of `ws_bytes`, or -1 when a layout of `bytes` does not fit.
int64_t sp_carve(uint64_t ws, uint64_t ws_bytes, uint64_t bytes) {
  char* o = carve((void*)(uintptr_t)ws, (size_t)ws_bytes, (size_t)bytes);
  return o ? (int64_t)((uintptr_t)o - (uintptr_t)ws) : -1;
}

}  // extern "C"
