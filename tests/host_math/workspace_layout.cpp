// TEST-ONLY: compiles kaolin_b200/csrc/workspace_layout.h as plain C++ (g++) so that
// tests/test_workspace_layout_cpu.py can check where every piece of the rasterizer's workspace
// lies, for any workspace pointer and size, on a CPU-only box.
#include <cstdint>
#include <cstddef>
#include "../../kaolin_b200/csrc/workspace_layout.h"

using namespace dibr_layout;

extern "C" {

// The carve of shape (B, NF, H, W, knum, f64) in the workspace (ws, ws_bytes).  out[0..5]: fits,
// origin, cache_tiles, min_bytes, tiles, bytes; then (at, bytes) of every piece in the order below;
// then the job counter's offset behind the records of `faces` faces for D = 1 .. kRowWalkMaxD.
int wl_carve(int B, int64_t NF, int H, int W, int knum, int f64, uint64_t ws, uint64_t ws_bytes,
             int64_t faces, int64_t* out) {
  const WorkspaceLayout L = workspace_layout({B, NF, H, W, knum, f64 != 0}, (const void*)(uintptr_t)ws, ws_bytes);
  const Piece pieces[] = {L.counters, L.cnt, L.pool_ctr, L.fb_ctr, L.band_ctr, L.view_flag, L.tile_cnt,
                          L.off, L.fb_list, L.band_list, L.entries, L.face_records,
                          L.xy, L.bbox_tight, L.bbox_large, L.valid, L.cache_hdr, L.cache_data};
  int n = 0;
  out[n++] = L.fits; out[n++] = (int64_t)L.origin; out[n++] = (int64_t)L.cache_tiles;
  out[n++] = (int64_t)L.min_bytes; out[n++] = (int64_t)L.tiles; out[n++] = (int64_t)L.bytes;
  for (const Piece& p : pieces) { out[n++] = (int64_t)p.at; out[n++] = (int64_t)p.bytes; }
  for (int D = 1; D <= kRowWalkMaxD; ++D) out[n++] = (int64_t)L.job_ctr(faces, D).at;
  return n;
}

}  // extern "C"
