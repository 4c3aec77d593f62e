// workspace_layout.h — where the rasterizer keeps its state in the caller's workspace.
//
// One function, workspace_layout, decides every piece's offset and size; the size queries of the
// C ABI, the scene setup of every entry point and the backward's face records all read it.  Plain
// C++ without CUDA, so that tests/host_math can compile it on a CPU and check each piece's place.
//
// Offsets are relative to the origin, the workspace pointer rounded up to kAlign; every piece
// starts on a multiple of kAlign, except the counters inside the first one:
//   counters: cnt [2][B][NB] int, pool_ctr, fb_ctr, band_ctr, view_flag [B], tile_cnt [tiles] |
//   off [2][B][NB] int | fb_list [tiles] int | band_list [tiles][kBandRec] int |
//   entries [2][4*NF] int4 | face_records [NF][<= face_record_floats(kRowWalkMaxD)] f32, job counter |
//   float64 calls: xy [NF][6] f32 | bbox_tight [NF] float4 | bbox_large [NF] float4 | valid [NF] u8 |
//   cache_hdr [cache_tiles] int4 | cache_data [cache_tiles][3][256*knum] u32
//
// Three invariants rest on this one layout:
//   1. A forward and a DIBR_B200_BINS_VALID backward of the same shape carve the same pieces out of
//      the same workspace: the backward reads the bins, work lists and hit cache the forward left.
//   2. The face records and the job counter, which the rasterize branch of a backward writes,
//      overlap no other piece: its soft-mask branch then reads the bins, work lists and hit cache.
//      Their room holds the records of every face at the largest D the row walk takes.
//   3. The memset before binning clears exactly `counters`, and every counter lies inside it.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "op_layouts.h"

namespace dibr_layout {

constexpr int kTile = 16;         // px per side of a screen tile, the finest bin
constexpr int kMaxLevels = 6;     // 16 * 4^5 = 16384 px
constexpr int kBandRec = 24;      // ints per record of the soft-mask work list
constexpr int kRowWalkMaxD = 4;   // the largest feature dim the row-walk rasterize backward takes
constexpr size_t kInt4Bytes = 4 * sizeof(int);

// Floats per face record of the row-walk backward: 6 vertex-gradient and 3*D feature sums, padded to float4.
constexpr int face_record_floats(int D) { return (6 + 3 * D + 3) & ~3; }

inline int levels_for(int H, int W) {
  int L = 1;
  while ((kTile << (2 * (L - 1))) < (H > W ? H : W)) ++L;
  return L;
}

inline int bins_per_view(int H, int W) {
  int nb = 0;
  const int L = levels_for(H, W);
  for (int l = 0; l < L; ++l) {
    const int t = kTile << (2 * l);
    nb += ((W + t - 1) / t) * ((H + t - 1) / t);
  }
  return nb;
}

struct LayoutShape {
  int B;          // views
  int64_t NF;     // faces in all views
  int H, W;
  int knum;       // > 0: a soft-mask hit cache
  bool f64;       // the float scene of a float64 call
};

struct WorkspaceLayout {
  size_t origin;     // carve: bytes from the workspace pointer to the origin
  bool fits;         // carve: the workspace is not null and holds min_bytes
  size_t tiles;      // 16x16 screen tiles in all views
  Piece counters, cnt, pool_ctr, fb_ctr, band_ctr, view_flag, tile_cnt;
  Piece off, fb_list, band_list, entries;
  Piece face_records;  // the row walk's records of up to NF faces with D <= kRowWalkMaxD, and its job counter
  Piece xy, bbox_tight, bbox_large, valid;
  Piece cache_hdr, cache_data;
  size_t cache_tiles;
  size_t min_bytes;  // every piece but the hit cache, from a pointer of any alignment
  size_t bytes;      // size query: min_bytes and the hit cache of cache_tiles tiles

  // The row walk's job counter, right behind the records of `faces` faces with D features: one
  // memset clears both.
  Piece job_ctr(int64_t faces, int D) const {
    return {face_records.at + (size_t)faces * face_record_floats(D) * sizeof(float), sizeof(int)};
  }
};

// Hit-cache data of one tile: 3 words per (pixel, hit).
inline size_t cache_tile_data_bytes(int knum) { return (size_t)3 * 256 * knum * sizeof(uint32_t); }

// The hit cache of n tiles at cache_hdr.at: a header {b, tx, ty, hits} per tile, then the tiles'
// data from the next kAlign.
inline void place_cache(WorkspaceLayout& L, size_t n, int knum) {
  L.cache_tiles = n;
  L.cache_hdr.bytes = n * kInt4Bytes;
  L.cache_data = {L.cache_hdr.at + align_up(L.cache_hdr.bytes, kAlign), n * cache_tile_data_bytes(knum)};
}

// Size query: the layout, with a hit cache of min(cache_tiles, tiles) tiles when knum > 0.
inline WorkspaceLayout workspace_layout(const LayoutShape& s, int64_t cache_tiles) {
  WorkspaceLayout L = {};
  const size_t nf = (size_t)(s.NF > 0 ? s.NF : 1);
  const size_t bins = (size_t)2 * s.B * bins_per_view(s.H, s.W);
  L.tiles = (size_t)((s.W + kTile - 1) / kTile) * ((s.H + kTile - 1) / kTile) * s.B;
  size_t at = 0;
  auto put = [&at](size_t bytes) {
    const Piece p = {at, bytes};
    at += align_up(bytes, kAlign);
    return p;
  };
  L.counters = put((bins + 3 + s.B + L.tiles) * sizeof(int));
  L.cnt = {0, bins * sizeof(int)};
  L.pool_ctr = {L.cnt.bytes, sizeof(int)};
  L.fb_ctr = {L.pool_ctr.at + sizeof(int), sizeof(int)};
  L.band_ctr = {L.fb_ctr.at + sizeof(int), sizeof(int)};
  L.view_flag = {L.band_ctr.at + sizeof(int), s.B * sizeof(int)};
  L.tile_cnt = {L.view_flag.at + L.view_flag.bytes, L.tiles * sizeof(int)};
  L.off = put(bins * sizeof(int));
  L.fb_list = put(L.tiles * sizeof(int));
  L.band_list = put(L.tiles * kBandRec * sizeof(int));
  L.entries = put((size_t)2 * 4 * nf * kInt4Bytes);
  L.face_records = put(nf * face_record_floats(kRowWalkMaxD) * sizeof(float) + sizeof(int));
  L.min_bytes = at + kAlign;   // up to kAlign - 1 bytes go to rounding the pointer up to the origin
  if (s.f64) {                 // the float64 pieces follow the float32 minimum
    at = L.min_bytes;
    L.xy = put(nf * 6 * sizeof(float));
    L.bbox_tight = put(nf * 4 * sizeof(float));
    L.bbox_large = put(nf * 4 * sizeof(float));
    L.valid = put(nf);
    L.min_bytes = at + kAlign;
  }
  size_t n = s.knum > 0 ? (size_t)cache_tiles : 0;
  if (n > L.tiles) n = L.tiles;
  L.cache_hdr.at = at;
  place_cache(L, n, s.knum);
  L.bytes = L.min_bytes;
  // one kAlign covers the rounding up of the cache header, and one more is spare
  if (s.knum > 0) L.bytes += 2 * kAlign + L.cache_hdr.bytes + L.cache_data.bytes;
  return L;
}

// Carve of the workspace (ws, ws_bytes): the pieces at origin + at, valid when `fits`.  With knum > 0
// the hit cache takes as many tiles, up to all of them, as the rest of the workspace holds.
inline WorkspaceLayout workspace_layout(const LayoutShape& s, const void* ws, size_t ws_bytes) {
  WorkspaceLayout L = workspace_layout(s, 0);
  L.origin = origin_offset(ws);
  L.fits = fits(ws, ws_bytes, L.min_bytes);
  if (L.fits && s.knum > 0) {
    const size_t room = ws_bytes - L.origin;   // from the origin to the workspace's end
    size_t n = (room - L.cache_hdr.at) / (kInt4Bytes + cache_tile_data_bytes(s.knum));
    if (n > L.tiles) n = L.tiles;
    place_cache(L, n, s.knum);
    while (n > 0 && L.cache_data.at + L.cache_data.bytes > room) place_cache(L, --n, s.knum);
  }
  return L;
}

}  // namespace dibr_layout
