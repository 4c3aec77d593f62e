"""kaolin.ops.conversions.marching_tetrahedra on sm_90a kernels (csrc/mesh_topology.cu), and
``MarchingTetrahedra``, which builds the grid's topology once.

The reference (tetmesh.py:57-168) rebuilds the grid's edges with ``torch.unique`` for every view of
every call and then makes about ten boolean-mask gathers, each a host synchronisation.  The grid does
not change between DMTet steps, so here its topology (the unique edges, each tet's six edge ids and the
adjacency) is built once; every call then flags each (view, edge) and classifies each (view, tet) in
one kernel, scans the flags once for all views, reads the per-view counts back (the call's one
device-to-host read) and writes every view's vertices and faces in one kernel each::

    M = MarchingTetrahedra(V, tets)           # once per grid
    verts, faces = M(vertices, sdf)           # per step, with autograd to vertices and sdf

An output vertex is a grid edge (a, b), a < b, whose ends are on either side of the surface
(sdf > 0 on exactly one; 0 and NaN count as outside), so the vertices of a view are its sign-change
edges in lexicographic order, as the reference's ``unique`` leaves them.
"""
import torch

from ... import _lib
from ..mesh import _TetTopology, _check

__all__ = ["marching_tetrahedra", "MarchingTetrahedra"]


def case_table():
    """(16, 2, 3, 2) int32: for each case sum_k occ(corner k) 2^k, the corner pairs (i, j) whose edges
    hold the vertices of each triangle, in the reference's order; -1 past the case's triangles."""
    return torch.tensor(_lib.marching_tets_case_table(), dtype=torch.int32).view(16, 2, 3, 2)


class _March(torch.autograd.Function):
    """x (B, V, 3), s (B, V) -> the vertices of every view in one (sum nv, 3) tensor; fills the faces
    (and tet indices) from the scan of the count pass."""

    @staticmethod
    def forward(ctx, x, s, topo, scan, num_vertices, faces, tet_idx):
        ctx.set_materialize_grads(False)
        B, V, E, T = x.shape[0], topo.num_vertices, topo.num_edges, topo.num_tets
        dev = x.device
        verts = torch.empty((num_vertices, 3), dtype=torch.float32, device=dev)
        vid = torch.empty(max(B * E, 1), dtype=torch.int32, device=dev)
        dummy = _lib.scratch(16, dev)      # for outputs with no rows, whose pointers would be NULL
        _lib.call("dibr_b200_marching_tets_emit", dev,
                  B, V, E, T, topo.edges, topo.tets, topo.tet_edge, x, s, scan, vid,
                  verts if num_vertices else dummy, faces if faces.numel() else dummy,
                  None if tet_idx is None else tet_idx if tet_idx.numel() else dummy, what="marching_tetrahedra")
        ctx.topo, ctx.num_vertices = topo, num_vertices
        ctx.save_for_backward(x, s, vid)
        return verts

    @staticmethod
    def backward(ctx, grad):
        x, s, vid = ctx.saved_tensors
        want_x, want_s = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if grad is None or not (want_x or want_s):
            return None, None, None, None, None, None, None
        if ctx.num_vertices == 0:
            return (torch.zeros_like(x) if want_x else None, torch.zeros_like(s) if want_s else None,
                    None, None, None, None, None)
        topo = ctx.topo
        gx = torch.empty_like(x) if want_x else None
        gs = torch.empty_like(s) if want_s else None
        _lib.call("dibr_b200_marching_tets_backward", x.device,
                  x.shape[0], topo.num_vertices, topo.num_edges, topo.adj_ptr, topo.adj, topo.adj_edge, x, s, vid,
                  grad.contiguous(), gx, gs, what="marching_tetrahedra")
        return gx, gs, None, None, None, None, None


class MarchingTetrahedra:
    r"""Marching tetrahedra on one tet grid, its topology built once.

    ``M = MarchingTetrahedra(num_vertices, tets)`` builds the grid's edges and adjacency;
    ``M(vertices, sdf, return_tet_idx=False)`` then returns what
    ``marching_tetrahedra(vertices, tets, sdf, return_tet_idx)`` returns, with autograd to
    ``vertices`` (B, num_vertices, 3) and ``sdf`` (B, num_vertices), float32, contiguous or not.  A
    call makes one device-to-host read (the per-view counts, which size the outputs); its backward
    makes none and uses no atomics, so results are bit-reproducible.
    """

    def __init__(self, num_vertices, tets):
        self._topo = _TetTopology("MarchingTetrahedra", num_vertices, tets)
        self.num_vertices = self._topo.num_vertices
        self.tets = self._topo.tets

    def __call__(self, vertices, sdf, return_tet_idx=False):
        func = "MarchingTetrahedra"
        topo = self._topo
        _check(func, [("vertices", vertices, torch.float32), ("sdf", sdf, torch.float32),
                      ("tets", topo.tets, torch.int64)])
        V = topo.num_vertices
        if vertices.dim() != 3 or tuple(vertices.shape[1:]) != (V, 3):
            raise RuntimeError(f"{func}: expected vertices of shape (B, {V}, 3), got {list(vertices.shape)}")
        B = vertices.shape[0]
        if tuple(sdf.shape) != (B, V):
            raise RuntimeError(f"{func}: expected sdf of shape ({B}, {V}), got {list(sdf.shape)}")
        if B == 0:
            return []
        E, T = topo.num_edges, topo.num_tets
        dev = vertices.device
        nbytes = _lib.lib().dibr_b200_marching_tets_workspace_bytes(B, E, T)
        if nbytes == 0:
            raise RuntimeError(f"{func}: {B} views of {E} edges and {T} tets do not fit 32-bit indices")
        x, s = vertices.contiguous(), sdf.contiguous()
        scan = torch.empty(B * (E + 2 * T) + 1, dtype=torch.int32, device=dev)
        counts = torch.empty((B, 3), dtype=torch.int32, device=dev)
        _lib.call("dibr_b200_marching_tets_count", dev,
                  B, V, E, T, topo.edges, topo.tets, s, scan, counts, _lib.scratch(nbytes, dev), nbytes,
                  what="marching_tetrahedra")
        counts = counts.tolist()                          # the call's one device-to-host read
        nv = [c[0] for c in counts]
        nf = [c[1] + 2 * c[2] for c in counts]
        i64 = dict(dtype=torch.int64, device=dev)
        faces = torch.empty((sum(nf), 3), **i64)
        tet_idx = torch.empty(sum(nf), **i64) if return_tet_idx else None
        verts = _March.apply(x, s, topo, scan, sum(nv), faces, tet_idx)
        out = [torch.split(verts, nv), torch.split(faces, nf)]
        if return_tet_idx:
            out.append(torch.split(tet_idx, nf))
        return out


def marching_tetrahedra(vertices, tets, sdf, return_tet_idx=False):
    r"""kaolin.ops.conversions.marching_tetrahedra: the triangle mesh of the zero level set of ``sdf``
    (B, V) on the tet grid (``vertices`` (B, V, 3), ``tets`` (T, 4)), per view.

    Returns ``[verts, faces]`` or ``[verts, faces, tet_idx]``, each a tuple of B tensors: vertices
    (nv, 3) float32, faces (nf, 3) int64 and the tet of each face (nf,) int64, bit-equal to the
    reference.  B = 0 returns ``[]``; no tets or no surface gives (0, 3) tensors.  The function builds
    the grid's topology on every call; ``MarchingTetrahedra`` builds it once.  That build sorts the
    adjacency of the whole grid, which costs far more than one call (116 ms against 0.9 ms for
    12.6 M tets on an H100; DESIGN.md §7 f10), so a training loop should build the class once.

    Deliberate deviations: only float32 vertices and sdf and int64 tets are accepted (the reference
    takes any float dtype and int32 tets); a tet index outside [0, V) raises ``IndexError``.
    """
    func = "marching_tetrahedra"
    _check(func, [("vertices", vertices, torch.float32), ("tets", tets, torch.int64)])
    if vertices.dim() != 3:
        raise RuntimeError(f"{func}: expected vertices of shape (B, V, 3), got {list(vertices.shape)}")
    return MarchingTetrahedra(vertices.shape[1], tets)(vertices, sdf, return_tet_idx)
