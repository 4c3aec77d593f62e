// op_layouts.h — where every operator outside the rasterizer keeps its scratch in the caller's workspace.
//
// One function per operator family returns its pieces and its total; the family's size query returns
// that total and its entry points carve with the same function, so the two cannot disagree.  Plain
// C++ without CUDA, so that tests/host_math can compile it on a CPU and check each piece's place.
//
// Every family follows one rule (the rasterizer's workspace_layout.h uses the same origin and fit):
//   - pieces go back to back from the origin, each starting on a multiple of kAlign;
//   - the origin is the workspace pointer rounded up to kAlign, so a workspace of any alignment works;
//   - the total is the end of the last piece plus kAlign, which covers that rounding; the workspace
//     fits when it is not NULL and holds the total.
// A memset that clears several counters clears one piece that holds them all.
#pragma once
#include <stddef.h>
#include <stdint.h>

namespace dibr_layout {

constexpr size_t kAlign = 256;
constexpr int kScanTile = 4096;   // elements per CTA of the exclusive scan (scan.cuh)
constexpr int kMaxCells = 16;     // grid cells a face may be inserted in; wider faces go to the view's wide list

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct Piece { size_t at, bytes; };

// Places pieces back to back, each rounded up to kAlign; total() adds kAlign of slack for the origin.
struct Placer {
  size_t at = 0, end = 0;
  Piece put(size_t bytes) {
    const Piece p = {at, bytes};
    end = at + bytes;
    at += align_up(bytes, kAlign);
    return p;
  }
  size_t total() const { return end + kAlign; }
};

// Bytes from the workspace pointer to the origin.
inline size_t origin_offset(const void* ws) {
  const uintptr_t p = (uintptr_t)ws;
  return align_up(p, kAlign) - p;
}

inline bool fits(const void* ws, size_t ws_bytes, size_t bytes) { return ws && ws_bytes >= bytes; }

// The origin of a workspace that fits a layout of `bytes`, or NULL.
inline char* carve(void* ws, size_t ws_bytes, size_t bytes) {
  return fits(ws, ws_bytes, bytes) ? (char*)ws + origin_offset(ws) : nullptr;
}

template <typename T>
T* piece(char* origin, Piece p) { return reinterpret_cast<T*>(origin + p.at); }

// The exclusive scan's tile sums for n elements (one int per tile and one spare).
inline size_t scan_sums_bytes(int64_t n) { return sizeof(int) * (size_t)((n + kScanTile - 1) / kScanTile + 1); }

// ---------------------------------------------------------------------------------------------
// The per-view face grid of grid_bins.cuh, shared by DefTet and the check_sign build.

// G x G cells for F faces per view: about one face per cell before overlaps.
inline int grid_side(int F) {
  int G = 8;
  while (G < 256 && (int64_t)G * G < F) G += 8;
  return G;
}

// counters holds cnt and off, [B][G*G + 1] int each and each from a multiple of kAlign: the check_sign
// build clears both with one memset.
struct GridBins { Piece bounds, counters, cnt, off, entries, wide; };

inline GridBins grid_bins(Placer& p, int B, int F) {
  const size_t G = (size_t)grid_side(F), nf = (size_t)B * (size_t)(F > 0 ? F : 1);
  const size_t cells = (size_t)B * (G * G + 1) * sizeof(int), room = align_up(cells, kAlign);
  GridBins g;
  g.bounds = p.put((size_t)B * 4 * sizeof(float));
  g.counters = p.put(2 * room);
  g.cnt = {g.counters.at, cells};
  g.off = {g.counters.at + room, cells};
  g.entries = p.put(nf * kMaxCells * sizeof(int));
  g.wide = p.put(nf * sizeof(int));
  return g;
}

struct DeftetLayout { GridBins grid; size_t bytes; };

inline DeftetLayout deftet_layout(int B, int F) {
  Placer p;
  DeftetLayout L;
  L.grid = grid_bins(p, B, F);
  L.bytes = p.total();
  return L;
}

// The check_sign build ("mesh"), which its queries read: the normalising scale maxlen [B] T, the grid,
// the face boxes [B][F] float4 and the face records [B][F][9] T, for T of tsize bytes.
struct CheckSignBuildLayout { Piece maxlen; GridBins grid; Piece boxes, records; size_t bytes; };

inline CheckSignBuildLayout check_sign_build_layout(int B, int F, size_t tsize) {
  const size_t nf = (size_t)B * (size_t)(F > 0 ? F : 1);
  Placer p;
  CheckSignBuildLayout L;
  L.maxlen = p.put((size_t)B * tsize);
  L.grid = grid_bins(p, B, F);
  L.boxes = p.put(nf * 4 * sizeof(float));
  L.records = p.put(nf * 9 * tsize);
  L.bytes = p.total();
  return L;
}

// A check_sign query of N points per view: the points binned on the build's grid (cnt, off as in the
// grid) and each point's cell and place in cell order.
struct CheckSignQueryLayout { Piece cnt, off, pcell, order; size_t bytes; };

inline CheckSignQueryLayout check_sign_query_layout(int B, int F, int N) {
  const size_t G = (size_t)grid_side(F), np = (size_t)B * (size_t)(N > 0 ? N : 1);
  const size_t cells = (size_t)B * (G * G + 1) * sizeof(int);
  Placer p;
  CheckSignQueryLayout L;
  L.cnt = p.put(cells);
  L.off = p.put(cells);
  L.pcell = p.put(np * sizeof(int));
  L.order = p.put(np * sizeof(int));
  L.bytes = p.total();
  return L;
}

// ---------------------------------------------------------------------------------------------
// mesh_topology.cu

// The CSR build of V vertices and `corners` corners with R raw neighbours each: per-vertex counts, the
// raw neighbours, the scan's tile sums, the long-row list and its counter.
struct TopoPieces { Piece count, raw, sums, long_rows, long_count; };

inline TopoPieces topo_pieces(Placer& p, int V, int64_t corners, int R) {
  TopoPieces t;
  t.count = p.put(sizeof(int) * (size_t)V);
  t.raw = p.put(sizeof(int) * (size_t)R * (size_t)corners);
  t.sums = p.put(scan_sums_bytes(V));
  t.long_rows = p.put(sizeof(int) * (size_t)V);
  t.long_count = p.put(sizeof(int));
  return t;
}

struct MeshTopologyLayout { TopoPieces topo; size_t bytes; };

inline MeshTopologyLayout mesh_topology_layout(int V, int64_t F, int S) {
  Placer p;
  MeshTopologyLayout L;
  L.topo = topo_pieces(p, V, F * S, 2);
  L.bytes = p.total();
  return L;
}

// Loop subdivision's edge numbering: per-vertex counts and the scan's tile sums.
struct SubdivisionLayout { Piece count, sums; size_t bytes; };

inline SubdivisionLayout subdivision_layout(int V) {
  Placer p;
  SubdivisionLayout L;
  L.count = p.put(sizeof(int) * (size_t)V);
  L.sums = p.put(scan_sums_bytes(V));
  L.bytes = p.total();
  return L;
}

// The tet-mesh topology: the CSR build of T tets (R = 3), then the corner CSR, degrees, weights and the
// build's two status words, which the caller does not keep, and the edge offsets [V + 1].
struct TetTopologyLayout { TopoPieces topo; Piece corner_ptr, corners, degree, weight, status, edge_ptr; size_t bytes; };

inline TetTopologyLayout tet_topology_layout(int V, int64_t T) {
  Placer p;
  TetTopologyLayout L;
  L.topo = topo_pieces(p, V, 4 * T, 3);
  L.corner_ptr = p.put(sizeof(int) * ((size_t)V + 1));
  L.corners = p.put(sizeof(int) * 4 * (size_t)T);
  L.degree = p.put(sizeof(int) * (size_t)V);
  L.weight = p.put(sizeof(float) * (size_t)V);
  L.status = p.put(2 * sizeof(int));
  L.edge_ptr = p.put(sizeof(int) * ((size_t)V + 1));
  L.bytes = p.total();
  return L;
}

// Marching tets: one flag per (view, edge) and two per (view, tet), and the scan's tile sums.
struct MarchingTetsLayout { Piece flags, sums; size_t bytes; };

inline MarchingTetsLayout marching_tets_layout(int B, int E, int64_t T) {
  const int64_t n = (int64_t)B * (E + 2 * T);
  Placer p;
  MarchingTetsLayout L;
  L.flags = p.put(sizeof(int) * (size_t)n);
  L.sums = p.put(scan_sums_bytes(n));
  L.bytes = p.total();
  return L;
}

// ---------------------------------------------------------------------------------------------
// marching_cubes.cu: the triangle and owned-vertex counts of `cubes` cubes (all views), one after the
// other, and the scan's tile sums.
struct MarchingCubesLayout { Piece counts, sums; size_t bytes; };

inline MarchingCubesLayout marching_cubes_layout(int64_t cubes) {
  Placer p;
  MarchingCubesLayout L;
  L.counts = p.put(2 * sizeof(int) * (size_t)cubes);
  L.sums = p.put(scan_sums_bytes(cubes));
  L.bytes = p.total();
  return L;
}

// ---------------------------------------------------------------------------------------------
// cubic_meshes.cu, for `batch` views of `lattice` corner points each.  Each view's lattice is
// padded to kCmWordBits-point words, `cubic_meshes_words(lattice)` per view and plane.  Seven bit
// planes [7][batch words]: the face planes x, y, z and the corner plane in the order the scan reads
// them, then the three reversal planes; the scan's input (one popcount per scanned word) and its
// output [4 batch words + 1]; the scan's tile sums.  Everything lives from the count call to the
// emit call.
constexpr int kCmWordBits = 32;

inline int64_t cubic_meshes_words(int64_t lattice) { return (lattice + kCmWordBits - 1) / kCmWordBits; }

struct CubicMeshesLayout { Piece bits, counts, scan, sums; size_t bytes; };

inline CubicMeshesLayout cubic_meshes_layout(int64_t batch, int64_t lattice) {
  const int64_t n = 4 * batch * cubic_meshes_words(lattice);   // scanned words
  Placer p;
  CubicMeshesLayout L;
  L.bits = p.put(sizeof(uint32_t) * (size_t)(n / 4 * 7));
  L.counts = p.put(sizeof(int) * (size_t)n);
  L.scan = p.put(sizeof(int) * ((size_t)n + 1));
  L.sums = p.put(scan_sums_bytes(n));
  L.bytes = p.total();
  return L;
}

// ---------------------------------------------------------------------------------------------
// point_mesh_distance.cu, for B views of N points and F faces, T of tsize bytes.
// Forward: one record of kFaceRecord T per (view, face) and one 64-bit search key per (view, point).
// Backward: the nine face terms per (view, point), then the points grouped by (view, closest face):
// counts [B*F], offsets [B*F + 1], the scan's tile sums, the point ids [B*N], the long-row list
// [B*F] and its counter.
constexpr int kFaceRecord = 33;   // v1, v2, v3, e12, e23, e31, three edge normals, unit normal, |e|^2 x 3

struct PointMeshForwardLayout { Piece records, keys; size_t bytes; };

inline PointMeshForwardLayout point_mesh_forward_layout(int B, int N, int F, size_t tsize) {
  const size_t nf = (size_t)B * (size_t)(F > 0 ? F : 1), np = (size_t)B * (size_t)(N > 0 ? N : 1);
  Placer p;
  PointMeshForwardLayout L;
  L.records = p.put(nf * kFaceRecord * tsize);
  L.keys = p.put(np * sizeof(unsigned long long));
  L.bytes = p.total();
  return L;
}

struct PointMeshBackwardLayout { Piece terms, count, off, sums, ids, long_rows, long_count; size_t bytes; };

inline PointMeshBackwardLayout point_mesh_backward_layout(int B, int N, int F, size_t tsize) {
  const int64_t nf = (int64_t)B * F;
  const size_t np = (size_t)B * (size_t)(N > 0 ? N : 1);
  Placer p;
  PointMeshBackwardLayout L;
  L.terms = p.put(np * 9 * tsize);
  L.count = p.put(sizeof(int) * (size_t)(nf > 0 ? nf : 1));
  L.off = p.put(sizeof(int) * ((size_t)nf + 1));
  L.sums = p.put(scan_sums_bytes(nf));
  L.ids = p.put(np * sizeof(int));
  L.long_rows = p.put(sizeof(int) * (size_t)(nf > 0 ? nf : 1));
  L.long_count = p.put(sizeof(int));
  L.bytes = p.total();
  return L;
}

// ---------------------------------------------------------------------------------------------
// voxelize.cu: the bit grid of `nwords` 32-bit words, the work items of `faces` (view, face) pairs and
// their exclusive scan, the set bits of each chunk of 32 words and their exclusive scan, and the tile
// sums of whichever scan is longer (the two run one after the other).
struct VoxelizeLayout { Piece bits, counts, scan, chunk_counts, chunk_scan, sums; size_t bytes; };

inline VoxelizeLayout voxelize_layout(int64_t nwords, int64_t faces, int64_t nchunks) {
  Placer p;
  VoxelizeLayout L;
  L.bits = p.put(sizeof(uint32_t) * (size_t)nwords);
  L.counts = p.put(sizeof(int) * (size_t)faces);
  L.scan = p.put(sizeof(int) * ((size_t)faces + 1));
  L.chunk_counts = p.put(sizeof(int) * (size_t)nchunks);
  L.chunk_scan = p.put(sizeof(int) * ((size_t)nchunks + 1));
  L.sums = p.put(scan_sums_bytes(faces > nchunks ? faces : nchunks));
  L.bytes = p.total();
  return L;
}

// ---------------------------------------------------------------------------------------------
// sample_points.cu, for B views of nf faces in all (packed or B x F), N samples per view, T of tsize
// bytes.  Forward: the float64 areas scanned in place into each view's CDF [nf], and per tile of
// kCdfTile faces the CDF at its last face (the coarse table), the tile's segmented sum and whether a
// view starts in it, and the carry from earlier tiles; one invalid-distribution flag per view.
// Backward: the per-corner vertex gradients [nf][3][3] T, then the samples grouped by face: counts
// [nf], offsets [nf + 1], the scan's tile sums, the sample ids [B*N], the long-row list [nf] and its
// counter.  face_areas' backward uses the corner gradients only.
constexpr int kCdfTile = 4096;

inline int64_t cdf_tiles(int64_t nf) { return (nf + kCdfTile - 1) / kCdfTile; }

struct SamplePointsForwardLayout { Piece cdf, coarse, tile_sum, tile_flag, carry, view_flag; size_t bytes; };

inline SamplePointsForwardLayout sample_points_forward_layout(int B, int64_t nf) {
  const size_t n = (size_t)(nf > 0 ? nf : 1), tiles = (size_t)(nf > 0 ? cdf_tiles(nf) : 1);
  Placer p;
  SamplePointsForwardLayout L;
  L.cdf = p.put(n * sizeof(double));
  L.coarse = p.put(tiles * sizeof(double));
  L.tile_sum = p.put(tiles * sizeof(double));
  L.tile_flag = p.put(tiles * sizeof(int));
  L.carry = p.put(tiles * sizeof(double));
  L.view_flag = p.put((size_t)(B > 0 ? B : 1) * sizeof(int));
  L.bytes = p.total();
  return L;
}

struct SamplePointsBackwardLayout { Piece corner_grad, count, off, sums, ids, long_rows, long_count; size_t bytes; };

inline SamplePointsBackwardLayout sample_points_backward_layout(int B, int64_t nf, int N, size_t tsize) {
  const size_t n = (size_t)(nf > 0 ? nf : 1), np = (size_t)B * (size_t)(N > 0 ? N : 1);
  Placer p;
  SamplePointsBackwardLayout L;
  L.corner_grad = p.put(n * 9 * tsize);
  L.count = p.put(n * sizeof(int));
  L.off = p.put((n + 1) * sizeof(int));
  L.sums = p.put(scan_sums_bytes(nf));
  L.ids = p.put((np > 0 ? np : 1) * sizeof(int));
  L.long_rows = p.put(n * sizeof(int));
  L.long_count = p.put(sizeof(int));
  L.bytes = p.total();
  return L;
}

// ---------------------------------------------------------------------------------------------
// voxelgrid.cu: fill's union-find labels, one int32 per voxel of `batch` views of `voxels` each.
struct VoxelgridFillLayout { Piece labels; size_t bytes; };

inline VoxelgridFillLayout voxelgrid_fill_layout(int64_t batch, int64_t voxels) {
  Placer p;
  VoxelgridFillLayout L;
  L.labels = p.put(sizeof(int32_t) * (size_t)batch * (size_t)voxels);
  L.bytes = p.total();
  return L;
}

// ---------------------------------------------------------------------------------------------
// pointcloud.cu: farthest point sampling of B views of N points, k rounds.
//
// A CTA of kFpsThreads threads keeps kFpsRegPoints points per thread in registers and, past that, up
// to kFpsSmemPoints per thread in shared memory (16 B each: x, y, z and the key).  A view goes to
// one thread-block cluster when it fits there: the cluster is the smallest that holds the view in
// registers, and only a view that needs more than max_cluster CTAs' registers also uses their
// shared memory.  Larger views take the grid path (one cooperative launch, a contiguous slice of a
// view per CTA); their points past a CTA's on-chip share live in the workspace.
//
// Workspace: the center's chunk sums [B][chunks] (sum x, y, z and the finite count as doubles, one
// chunk per kFpsChunk points), the centers [B] float4, and on the grid path the round slots
// [B][3] uint64 and a float4 (x, y, z, key) per point [B][N].
constexpr int kFpsThreads = 256;
constexpr int kFpsRegPoints = 32;
constexpr int kFpsSmemPoints = 48;
constexpr int kFpsChunk = 1024;
constexpr int64_t kFpsCtaRegs = (int64_t)kFpsThreads * kFpsRegPoints;                     // 8192
constexpr int64_t kFpsCtaOnChip = (int64_t)kFpsThreads * (kFpsRegPoints + kFpsSmemPoints);  // 20480

enum FpsPath { kFpsNothing = 0, kFpsCluster = 1, kFpsGrid = 2 };

// The cluster path's CTAs per view and shared-memory points per thread for a view of N points.
struct FpsPlan { int path, cluster, smem_points; };

// Shared-memory points per thread for a CTA that owns n points.
inline int fps_smem_points(int64_t n) {
  const int64_t extra = n - kFpsCtaRegs;
  if (extra <= 0) return 0;
  const int64_t q = (extra + kFpsThreads - 1) / kFpsThreads;
  return (int)(q < kFpsSmemPoints ? q : kFpsSmemPoints);
}

inline FpsPlan fps_plan(int64_t B, int64_t N, int64_t k, int max_cluster) {
  FpsPlan p = {kFpsNothing, 0, 0};
  if (B <= 0 || N <= 0 || k <= 0 || max_cluster <= 0) return p;
  const int64_t by_regs = (N + kFpsCtaRegs - 1) / kFpsCtaRegs;
  if (by_regs <= max_cluster) {
    p.path = kFpsCluster;
    p.cluster = (int)by_regs;
  } else if (N <= max_cluster * kFpsCtaOnChip) {
    p.path = kFpsCluster;
    p.cluster = max_cluster;
    p.smem_points = fps_smem_points((N + max_cluster - 1) / max_cluster);
  } else {
    p.path = kFpsGrid;
  }
  return p;
}

inline int64_t fps_chunks(int64_t N) { return (N + kFpsChunk - 1) / kFpsChunk; }

struct FpsLayout { FpsPlan plan; Piece chunk_sums, centers, slots, points; size_t bytes; };

inline FpsLayout fps_layout(int64_t B, int64_t N, int64_t k, int max_cluster) {
  FpsLayout L;
  L.plan = fps_plan(B, N, k, max_cluster);
  const size_t views = (size_t)(B > 0 ? B : 0), grid = L.plan.path == kFpsGrid;
  Placer p;
  L.chunk_sums = p.put(views * (size_t)fps_chunks(N > 0 ? N : 0) * 4 * sizeof(double));
  L.centers = p.put(views * 4 * sizeof(float));
  L.slots = p.put(grid * views * 3 * sizeof(uint64_t));
  L.points = p.put(grid * views * (size_t)N * 4 * sizeof(float));
  L.bytes = p.total();
  return L;
}

// ---------------------------------------------------------------------------------------------
// lighting.cu: the light gradients' partial sums, `floats` per light in each of `slots` CTA slots.
struct LightingLayout { Piece partial; size_t bytes; };

inline LightingLayout lighting_layout(int slots, int floats, int lights) {
  Placer p;
  LightingLayout L;
  L.partial = p.put((size_t)slots * (size_t)lights * (size_t)floats * sizeof(float));
  L.bytes = p.total();
  return L;
}

}  // namespace dibr_layout
