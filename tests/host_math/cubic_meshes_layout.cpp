// TEST-ONLY: compiles the cubic-meshes layout of kaolin_b200/csrc/op_layouts.h as plain C++ (g++) so that
// tests/test_cubic_meshes_cpu.py can check where its pieces lie, for any workspace pointer, on a CPU-only box.
#include <cstdint>
#include <cstddef>
#include "../../kaolin_b200/csrc/op_layouts.h"

using namespace dibr_layout;

extern "C" {

// out = {total, words per view and plane, then (at, bytes) of bits, counts, scan and sums}.
void cm_layout(int64_t batch, int64_t lattice, int64_t* out) {
  const CubicMeshesLayout L = cubic_meshes_layout(batch, lattice);
  out[0] = (int64_t)L.bytes;
  out[1] = cubic_meshes_words(lattice);
  const Piece p[4] = {L.bits, L.counts, L.scan, L.sums};
  for (int i = 0; i < 4; ++i) {
    out[2 + 2 * i] = (int64_t)p[i].at;
    out[3 + 2 * i] = (int64_t)p[i].bytes;
  }
}

// The offset of the origin from a workspace at `ws` of `ws_bytes`, or -1 when a layout of `bytes` does not fit.
int64_t cm_carve(uint64_t ws, uint64_t ws_bytes, uint64_t bytes) {
  char* o = carve((void*)(uintptr_t)ws, (size_t)ws_bytes, (size_t)bytes);
  return o ? (int64_t)((uintptr_t)o - (uintptr_t)ws) : -1;
}

}  // extern "C"
