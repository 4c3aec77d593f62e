// TEST-ONLY: compiles kaolin_b200/csrc/op_layouts.h as plain C++ (g++) so that
// tests/test_op_layouts_cpu.py can check where every piece of each operator's workspace lies, for any
// workspace pointer, on a CPU-only box.
#include <cstdint>
#include <cstddef>
#include <initializer_list>
#include "../../kaolin_b200/csrc/op_layouts.h"

using namespace dibr_layout;

namespace {

int put(int64_t* out, int n, const Piece& p) {
  out[n] = (int64_t)p.at;
  out[n + 1] = (int64_t)p.bytes;
  return n + 2;
}

int put_grid(int64_t* out, int n, const GridBins& g) {
  for (const Piece& p : {g.bounds, g.counters, g.cnt, g.off, g.entries, g.wide}) n = put(out, n, p);
  return n;
}

int put_topo(int64_t* out, int n, const TopoPieces& t) {
  for (const Piece& p : {t.count, t.raw, t.sums, t.long_rows, t.long_count}) n = put(out, n, p);
  return n;
}

}  // namespace

extern "C" {

// The layout of one family for the arguments a[]: out[0] = its total, then (at, bytes) of every piece
// in the order tests/test_op_layouts_cpu.py names them.  Returns the number of values written, or -1.
int ol_layout(int family, const int64_t* a, int64_t* out) {
  int n = 1;
  switch (family) {
    case 0: {
      const DeftetLayout L = deftet_layout((int)a[0], (int)a[1]);
      out[0] = (int64_t)L.bytes;
      return put_grid(out, n, L.grid);
    }
    case 1: {
      const CheckSignBuildLayout L = check_sign_build_layout((int)a[0], (int)a[1], (size_t)a[2]);
      out[0] = (int64_t)L.bytes;
      n = put(out, n, L.maxlen);
      n = put_grid(out, n, L.grid);
      n = put(out, n, L.boxes);
      return put(out, n, L.records);
    }
    case 2: {
      const CheckSignQueryLayout L = check_sign_query_layout((int)a[0], (int)a[1], (int)a[2]);
      out[0] = (int64_t)L.bytes;
      for (const Piece& p : {L.cnt, L.off, L.pcell, L.order}) n = put(out, n, p);
      return n;
    }
    case 3: {
      const MeshTopologyLayout L = mesh_topology_layout((int)a[0], a[1], (int)a[2]);
      out[0] = (int64_t)L.bytes;
      return put_topo(out, n, L.topo);
    }
    case 4: {
      const SubdivisionLayout L = subdivision_layout((int)a[0]);
      out[0] = (int64_t)L.bytes;
      n = put(out, n, L.count);
      return put(out, n, L.sums);
    }
    case 5: {
      const TetTopologyLayout L = tet_topology_layout((int)a[0], a[1]);
      out[0] = (int64_t)L.bytes;
      n = put_topo(out, n, L.topo);
      for (const Piece& p : {L.corner_ptr, L.corners, L.degree, L.weight, L.status, L.edge_ptr}) n = put(out, n, p);
      return n;
    }
    case 6: {
      const MarchingTetsLayout L = marching_tets_layout((int)a[0], (int)a[1], a[2]);
      out[0] = (int64_t)L.bytes;
      n = put(out, n, L.flags);
      return put(out, n, L.sums);
    }
    case 7: {
      const MarchingCubesLayout L = marching_cubes_layout(a[0]);
      out[0] = (int64_t)L.bytes;
      n = put(out, n, L.counts);
      return put(out, n, L.sums);
    }
    case 8: {
      const LightingLayout L = lighting_layout((int)a[0], (int)a[1], (int)a[2]);
      out[0] = (int64_t)L.bytes;
      return put(out, n, L.partial);
    }
  }
  return -1;
}

// The carve of the workspace (ws, ws_bytes) for a layout of `bytes`: the origin's offset from ws, or -1
// when the workspace does not fit.
int64_t ol_carve(uint64_t ws, uint64_t ws_bytes, uint64_t bytes) {
  char* p = (char*)(uintptr_t)ws;
  char* o = carve(p, ws_bytes, bytes);
  return o ? (int64_t)(o - p) : -1;
}

}  // extern "C"
