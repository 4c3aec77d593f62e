"""kaolin.ops.mesh drop-ins on sm_90a kernels (csrc/mesh_topology.cu): ``adjacency_matrix``,
``uniform_laplacian``, ``average_face_vertex_features`` and ``compute_vertex_normals`` with the
reference's signatures, and ``UniformLaplacian``, the Laplacian without its V x V matrix.

The reference builds a dense V x V matrix (mesh.py:78-151), which does not fit in memory beyond a few
ten thousand vertices.  Here the topology of ``faces`` is built once into two CSR structures (the
corners of each vertex, and its unique neighbours) and every product is a gather over them.  The
functional forms rebuild it on every call, as the reference rebuilds its matrix; ``UniformLaplacian``
builds it once::

    L = UniformLaplacian(V, faces)            # instead of L = uniform_laplacian(V, faces)
    loss = (L @ (vertices - vertices_init)).pow(2).mean()

Deliberate deviation: a face index outside [0, V) raises ``IndexError`` (the reference does not check).

Loop subdivision (trianglemesh.py:482-612) is built on the same topology: ``subdivide_trianglemesh``
has the reference's signature and builds every level on each call; ``LoopSubdivision`` builds them
once and applies them with autograd to the vertices and a learnable per-vertex alpha::

    S = LoopSubdivision(V, faces, 2)          # coarse-to-fine DIB-R, or DMTet's learnable alpha
    fine_vertices = S(vertices, alpha)        # fine faces: S.faces

``subdivide_tetmesh`` (tetmesh.py:85-181) refines a tet grid on the topology of its tets, which
marching tetrahedra (``kaolin_b200.ops.conversions``) shares.
"""
import torch

from .. import _lib
from ..render.mesh import _host

__all__ = ["adjacency_matrix", "uniform_laplacian", "compute_vertex_normals", "average_face_vertex_features",
           "UniformLaplacian", "subdivide_trianglemesh", "LoopSubdivision", "subdivide_tetmesh"]


def _check(func, typed):
    """(name, tensor, dtype) triples: CUDA tensors on one device, each of its dtype; no CPU path."""
    dev = _host.check_tensors(func, [(name, t) for name, t, _ in typed], dtype=None)
    for name, t, dtype in typed:
        if t.dtype != dtype:
            raise RuntimeError(f"\"{func}\" not implemented for '{str(t.dtype).replace('torch.', '')}' "
                               f"(kaolin_b200 takes {name} as {str(dtype).replace('torch.', '')})")
    return dev


class _Topology:
    """The corner and adjacency CSRs of one mesh (see include/dibr_b200.h).  With ``status`` (an int32
    CUDA tensor of at least 2 elements) the build writes its status there and the caller reads it and
    calls ``_finish``; otherwise the constructor reads it."""

    def __init__(self, func, num_vertices, faces, status=None):
        _check(func, [("faces", faces, torch.int64)])
        if faces.dim() != 2 or faces.shape[1] < 3:
            raise RuntimeError(f"{func}: expected faces of shape (num_faces, face_size >= 3), got {list(faces.shape)}")
        V, (F, S) = int(num_vertices), faces.shape
        if V < 0:
            raise ValueError(f"{func}: num_vertices must be >= 0, got {V}")
        nbytes = _lib.lib().dibr_b200_mesh_topology_workspace_bytes(V, F, S)
        if nbytes == 0:
            raise RuntimeError(f"{func}: {V} vertices or {F} faces of size {S} do not fit 32-bit indices")
        dev = faces.device
        faces = faces.contiguous()
        i32 = dict(dtype=torch.int32, device=dev)
        self.num_vertices, self.faces = V, faces
        self.corner_ptr = torch.empty(V + 1, **i32)
        self.corners = torch.empty(max(F * S, 1), **i32)      # never empty: the ABI takes no NULL buffers
        self.adj_ptr = torch.empty(V + 1, **i32)
        self._adj = torch.empty(max(2 * F * S, 1), **i32)
        self.degree = torch.empty(V, **i32)
        self.weight = torch.empty(V, dtype=torch.float32, device=dev)
        own = status is None
        if own:
            status = torch.empty(2, **i32)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _lib.call("dibr_b200_mesh_topology_build", dev,
                  V, F, S, faces, self.corner_ptr, self.corners, self.adj_ptr, self._adj, self.degree, self.weight,
                  status, ws, nbytes, what=func)
        if own:
            self._finish(func, *status.tolist())          # the build's one device-to-host read

    def _finish(self, func, edges, error):
        if error:
            raise IndexError(f"{func}: faces holds an index outside [0, {self.num_vertices})")
        self.num_edges = edges
        self.adj = self._adj[:edges]

    def apply(self, x, transpose, smooth):
        """(L or L^T, + I if smooth) applied to x (..., V, C) float32, on the current stream."""
        y = torch.empty_like(x)
        V, C = x.shape[-2], x.shape[-1]
        batch = x.numel() // max(V * C, 1)
        _lib.call("dibr_b200_laplacian_apply", x.device,
                  batch, V, C, self.adj_ptr, self._adj, self.weight, x, int(transpose), int(smooth), y,
                  what="laplacian_apply")
        return y

    def dense(self, laplacian):
        V = self.num_vertices
        out = torch.empty((V, V), dtype=torch.float32, device=self.faces.device)
        _lib.call("dibr_b200_mesh_dense", out.device, V, int(laplacian), self.adj_ptr, self._adj, self.weight, out,
                  what="uniform_laplacian" if laplacian else "adjacency_matrix")
        return out


class _Apply(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, topo, smooth):
        ctx.topo, ctx.smooth = topo, smooth
        return topo.apply(x, False, smooth)

    @staticmethod
    def backward(ctx, grad):
        return ctx.topo.apply(grad.contiguous(), True, ctx.smooth), None, None


def _apply(func, topo, x, smooth):
    _check(func, [("x", x, torch.float32), ("faces", topo.faces, torch.int64)])
    if x.dim() not in (2, 3) or x.shape[-2] != topo.num_vertices:
        raise RuntimeError(f"{func}: expected x of shape (V, k) or (B, V, k) with V = {topo.num_vertices}, "
                           f"got {list(x.shape)}")
    return _Apply.apply(x.contiguous(), topo, smooth)


class UniformLaplacian:
    r"""The uniform Laplacian of a mesh, built once, without its :math:`V \times V` matrix.

    ``L @ x`` (or ``L.matmul(x)``) equals ``torch.matmul(uniform_laplacian(num_vertices, faces), x)``
    for x of shape (V, k) or (B, V, k) float32, with autograd to x; ``L.to_dense()`` is
    ``uniform_laplacian(num_vertices, faces)``.  Memory is O(F·S + V).
    """

    def __init__(self, num_vertices, faces):
        self._topo = _Topology("UniformLaplacian", num_vertices, faces)

    def matmul(self, x):
        return _apply("UniformLaplacian.matmul", self._topo, x, False)

    __matmul__ = matmul

    def to_dense(self):
        return self._topo.dense(True)


def adjacency_matrix(num_vertices, faces, sparse=True):
    r"""kaolin.ops.mesh.adjacency_matrix: the (V, V) 0/1 adjacency, as a sparse COO tensor (indices in
    lexicographic order, not marked coalesced) or dense float32."""
    topo = _Topology("adjacency_matrix", num_vertices, faces)
    if not sparse:
        return topo.dense(False)
    E = topo.num_edges
    indices = torch.empty((2, E), dtype=torch.int64, device=faces.device)
    _lib.call("dibr_b200_adjacency_coo", faces.device, topo.num_vertices, E, topo.adj_ptr, topo._adj, indices,
              what="adjacency_matrix")
    values = torch.ones(E, dtype=torch.float32, device=faces.device)
    return torch.sparse_coo_tensor(indices, values, (topo.num_vertices, topo.num_vertices))


def uniform_laplacian(num_vertices, faces):
    r"""kaolin.ops.mesh.uniform_laplacian: the dense (V, V) float32 matrix, -1 on the diagonal and
    1 / num_neighbours(i) at the neighbours of i."""
    return _Topology("uniform_laplacian", num_vertices, faces).dense(True)


class _Average(torch.autograd.Function):
    @staticmethod
    def forward(ctx, face_features, topo):
        ctx.topo = topo
        B, F, S, N = face_features.shape
        V = topo.num_vertices
        out = torch.empty((B, V, N), dtype=torch.float32, device=face_features.device)
        _lib.call("dibr_b200_vertex_average_forward", out.device,
                  B, V, F, S, N, topo.corner_ptr, topo.corners, face_features, out, what="average_face_vertex_features")
        ctx.shape = face_features.shape
        return out

    @staticmethod
    def backward(ctx, grad):
        topo = ctx.topo
        B, F, S, N = ctx.shape
        grad = grad.contiguous()
        g_ff = torch.empty(ctx.shape, dtype=torch.float32, device=grad.device)
        _lib.call("dibr_b200_vertex_average_backward", grad.device,
                  B, topo.num_vertices, F, S, N, topo.faces, topo.corner_ptr, grad, g_ff,
                  what="average_face_vertex_features")
        return g_ff, None


def average_face_vertex_features(faces, face_features, num_vertices=None):
    r"""kaolin.ops.mesh.average_face_vertex_features: per-vertex mean of ``face_features``
    (B, F, S, N) float32 over the faces incident to each vertex -> (B, V, N); 0 where no face is."""
    func = "average_face_vertex_features"
    _check(func, [("face_features", face_features, torch.float32), ("faces", faces, torch.int64)])
    if faces.dim() != 2 or face_features.dim() != 4 or tuple(face_features.shape[1:3]) != tuple(faces.shape):
        raise RuntimeError(f"{func}: expected face_features of shape (B, {faces.shape[0]}, {faces.shape[-1]}, N), "
                           f"got {list(face_features.shape)}")
    if num_vertices is None:
        num_vertices = int(faces.max()) + 1
    topo = _Topology(func, num_vertices, faces)
    return _Average.apply(face_features.contiguous(), topo)


def compute_vertex_normals(faces, face_normals, num_vertices=None):
    r"""kaolin.ops.mesh.compute_vertex_normals: ``average_face_vertex_features`` of the per-corner
    normals (B, F, S, 3) -> (B, V, 3)."""
    return average_face_vertex_features(faces, face_normals, num_vertices=num_vertices)


class _SubdivisionLevel:
    """One level of Loop subdivision: the topology of (num_vertices, faces), its edges and the next
    level's faces (see include/dibr_b200.h), built with one device-to-host read, the edge count."""

    def __init__(self, func, num_vertices, faces):
        V, F = num_vertices, faces.shape[0]
        dev = faces.device
        status = torch.empty(3, dtype=torch.int32, device=dev)
        self.topo = _Topology(func, V, faces, status=status)
        nbytes = _lib.lib().dibr_b200_loop_subdivision_workspace_bytes(V, F)
        i32 = dict(dtype=torch.int32, device=dev)
        self.num_vertices, self.faces = V, self.topo.faces
        self.edge_ptr = torch.empty(V + 1, **i32)
        self.adj_edge = torch.empty(max(6 * F, 1), **i32)
        self.face_edge = torch.empty(max(3 * F, 1), **i32)
        self.edges = torch.empty((max(3 * F, 1), 4), **i32)
        self.new_faces = torch.empty((4 * F, 3), dtype=torch.int64, device=dev)
        ws = _lib.scratch(nbytes, dev)
        _lib.call("dibr_b200_loop_subdivision_build", dev,
                  V, F, self.faces, self.topo.corner_ptr, self.topo.corners,
                  self.topo.adj_ptr, self.topo._adj, self.edge_ptr, self.adj_edge, self.face_edge, self.edges,
                  self.new_faces, status[2:], ws, nbytes, what=func)
        adj_entries, error, E = status.tolist()          # the level's one device-to-host read
        self.topo._finish(func, adj_entries, error)
        self.num_edges = E


class _SubdivideStep(torch.autograd.Function):
    """One level applied to x (B, V, 3) and alpha (B, V) or None -> y (B, V + E, 3), plus the next
    level's alpha (B, V + E) when ``carry``."""

    @staticmethod
    def forward(ctx, x, alpha, level, carry):
        ctx.set_materialize_grads(False)
        t = level.topo
        B, V, E = x.shape[0], level.num_vertices, level.num_edges
        y = torch.empty((B, V + E, 3), dtype=torch.float32, device=x.device)
        a_out = torch.empty((B, V + E), dtype=torch.float32, device=x.device) if carry else None
        _lib.call("dibr_b200_loop_subdivision_forward", x.device,
                  B, V, E, t.adj_ptr, t._adj, level.edges, level.faces, x, alpha, y, a_out,
                  what="subdivide_trianglemesh")
        ctx.level, ctx.shape = level, x.shape
        need_alpha = alpha is not None and ctx.needs_input_grad[1]
        ctx.save_for_backward(x if need_alpha else None, alpha)
        return y if a_out is None else (y, a_out)

    @staticmethod
    def backward(ctx, grad, grad_alpha=None):
        x, alpha = ctx.saved_tensors
        level, t = ctx.level, ctx.level.topo
        B, V, _ = ctx.shape
        E = level.num_edges
        dev = level.faces.device
        if grad is None:
            grad = torch.zeros((B, V + E, 3), dtype=torch.float32, device=dev)
        gx = torch.empty(ctx.shape, dtype=torch.float32, device=dev) if ctx.needs_input_grad[0] else None
        ga = torch.empty((B, V), dtype=torch.float32, device=dev) if x is not None else None
        _lib.call("dibr_b200_loop_subdivision_backward", dev,
                  B, V, E, t.corner_ptr, t.corners, t.adj_ptr, t._adj, level.adj_edge, level.face_edge, level.edges,
                  x, alpha, grad.contiguous(), None if grad_alpha is None else grad_alpha.contiguous(), gx, ga,
                  what="subdivide_trianglemesh")
        return gx, ga, None, None


def _check_faces(func, faces):
    _check(func, [("faces", faces, torch.int64)])
    if faces.dim() != 2 or faces.shape[1] != 3:
        raise RuntimeError(f"{func}: expected triangle faces of shape (num_faces, 3), got {list(faces.shape)}")


class LoopSubdivision:
    r"""Loop subdivision of one triangle mesh, every level built once.

    ``S = LoopSubdivision(num_vertices, faces, iterations)`` builds the topology and the edges of
    every level; ``S(vertices, alpha=None)`` then computes
    ``subdivide_trianglemesh(vertices, faces, iterations, alpha)[0]`` with autograd to ``vertices``
    and ``alpha`` and no host synchronisation, and ``S.faces`` is the final
    :math:`(F \cdot 4^\text{iterations}, 3)` faces.  ``vertices`` (B, num_vertices, 3) and
    ``alpha`` (B, num_vertices) are float32 for any B.  Each level is one kernel forward and one
    backward; no floating-point atomics, so results are bit-reproducible.
    """

    def __init__(self, num_vertices, faces, iterations):
        func = "LoopSubdivision"
        _check_faces(func, faces)
        V, iterations = int(num_vertices), int(iterations)
        if V < 0 or iterations < 0:
            raise ValueError(f"{func}: num_vertices and iterations must be >= 0, got {V} and {iterations}")
        self.num_vertices, self.iterations = V, iterations
        self._levels = []
        f = faces.contiguous() if iterations else faces
        for _ in range(iterations):
            if _lib.lib().dibr_b200_loop_subdivision_workspace_bytes(V, f.shape[0]) == 0:
                raise RuntimeError(f"{func}: {V} vertices or {f.shape[0]} faces do not fit 32-bit indices")
            level = _SubdivisionLevel(func, V, f)
            self._levels.append(level)
            V, f = V + level.num_edges, level.new_faces
        self.faces = f
        self.num_output_vertices = V

    def __call__(self, vertices, alpha=None):
        func = "LoopSubdivision"
        typed = [("vertices", vertices, torch.float32), ("faces", self.faces, torch.int64)]
        if alpha is not None:
            typed.append(("alpha", alpha, torch.float32))
        _check(func, typed)
        V = self.num_vertices
        if vertices.dim() != 3 or vertices.shape[1:] != (V, 3):
            raise RuntimeError(f"{func}: expected vertices of shape (B, {V}, 3), got {list(vertices.shape)}")
        if alpha is not None and tuple(alpha.shape) != (vertices.shape[0], V):
            raise RuntimeError(f"{func}: expected alpha of shape ({vertices.shape[0]}, {V}), got {list(alpha.shape)}")
        if not self._levels:
            return vertices
        x = vertices.contiguous()
        a = None if alpha is None else alpha.contiguous()
        for k, level in enumerate(self._levels):
            carry = a is not None and k + 1 < len(self._levels)
            out = _SubdivideStep.apply(x, a, level, carry)
            x, a = out if carry else (out, None)
        return x


def subdivide_trianglemesh(vertices, faces, iterations, alpha=None):
    r"""kaolin.ops.mesh.subdivide_trianglemesh: ``iterations`` levels of Loop subdivision of
    ``vertices`` (B, V, 3) float32 with the unbatched ``faces`` (F, 3) int64 -> (vertices
    (B, V', 3), faces (F·4^iterations, 3)).  ``alpha`` (B, V) float32, if given, is the per-vertex
    smoothing weight (with autograd), carried to the new vertices from level to level as the
    reference does; otherwise each level uses Loop's weights.  The reference's quirks are kept: a vertex
    referenced by no face (and every vertex when F = 0) comes out NaN, whatever alpha is;
    ``iterations = 0`` returns the inputs.  The topology is built on every call, as the reference
    does; ``LoopSubdivision`` builds it once.

    Deliberate deviations: any B works (the reference raises for B > 1) and a given alpha must be
    (B, V); a face index outside [0, V) raises ``IndexError``; faces that are not triangles raise (the
    reference mis-indexes them); only float32 is accepted (the reference's buffers are float32).
    """
    func = "subdivide_trianglemesh"
    _check_faces(func, faces)
    _check(func, [("vertices", vertices, torch.float32), ("faces", faces, torch.int64)])
    if vertices.dim() != 3 or vertices.shape[-1] != 3:
        raise RuntimeError(f"{func}: expected vertices of shape (B, V, 3), got {list(vertices.shape)}")
    if int(iterations) == 0:
        if alpha is not None:
            _check(func, [("alpha", alpha, torch.float32), ("faces", faces, torch.int64)])
        return vertices, faces
    S = LoopSubdivision(vertices.shape[1], faces, iterations)
    return S(vertices, alpha), S.faces


def _trim(t, n):
    """The first n rows of a capacity-sized build output, as their own allocation (at least one row, so
    its pointer is never NULL)."""
    return t[:max(int(n), 1)].clone()


class _TetTopology:
    """The topology of a tet mesh (see include/dibr_b200.h): the adjacency CSR with all six edges of
    every tet, the unique edges (E, 2), each adjacency entry's edge id and each tet's six edge ids, built
    with one device-to-host read.  Shared by ``subdivide_tetmesh`` and marching tetrahedra."""

    def __init__(self, func, num_vertices, tets):
        _check(func, [("tets", tets, torch.int64)])
        if tets.dim() != 2 or tets.shape[1] != 4:
            raise RuntimeError(f"{func}: expected tets of shape (num_tets, 4), got {list(tets.shape)}")
        V, T = int(num_vertices), tets.shape[0]
        if V < 0:
            raise ValueError(f"{func}: num_vertices must be >= 0, got {V}")
        nbytes = _lib.lib().dibr_b200_tet_topology_workspace_bytes(V, T)
        if nbytes == 0:
            raise RuntimeError(f"{func}: {V} vertices or {T} tets do not fit 32-bit indices")
        dev = tets.device
        tets = tets.contiguous()
        i32 = dict(dtype=torch.int32, device=dev)
        adj_ptr = torch.empty(V + 1, **i32)
        adj = torch.empty(max(12 * T, 1), **i32)
        edges = torch.empty((max(6 * T, 1), 2), **i32)
        adj_edge = torch.empty(max(12 * T, 1), **i32)
        tet_edge = torch.empty((max(T, 1), 6), **i32)
        status = torch.empty(3, **i32)
        ws = _lib.scratch(nbytes, dev)
        _lib.call("dibr_b200_tet_topology_build", dev,
                  V, T, tets, adj_ptr, adj, edges, adj_edge, tet_edge, status, ws, nbytes, what=func)
        E, error, entries = status.tolist()              # the build's one device-to-host read
        if error:
            raise IndexError(f"{func}: tets holds an index outside [0, {V})")
        self.num_vertices, self.num_tets, self.num_edges, self.tets = V, T, E, tets
        self.adj_ptr, self.tet_edge = adj_ptr, tet_edge
        self.adj, self.adj_edge, self.edges = _trim(adj, entries), _trim(adj_edge, entries), _trim(edges, E)


class _TetSubdivide(torch.autograd.Function):
    """x (B, V, 3) and f (B, V, D) -> (y (B, V + E, 3), yf (B, V + E, D)); fills new_tets (8T, 4)."""

    @staticmethod
    def forward(ctx, x, f, topo, new_tets):
        ctx.set_materialize_grads(False)
        B, V, D = x.shape[0], topo.num_vertices, f.shape[-1]
        E = topo.num_edges
        y = torch.empty((B, V + E, 3), dtype=torch.float32, device=x.device)
        yf = torch.empty((B, V + E, D), dtype=torch.float32, device=x.device)
        _lib.call("dibr_b200_tet_subdivide_forward", x.device,
                  B, V, E, topo.num_tets, D, topo.edges, topo.tets, topo.tet_edge, x, f if D else None, y,
                  yf if D else None, new_tets, what="subdivide_tetmesh")
        ctx.topo, ctx.shape = topo, (B, V, D)
        return y, yf

    @staticmethod
    def backward(ctx, gy, gyf):
        topo = ctx.topo
        B, V, D = ctx.shape
        dev = topo.tets.device
        gx = torch.empty((B, V, 3), dtype=torch.float32, device=dev) if ctx.needs_input_grad[0] and gy is not None else None
        gf = (torch.empty((B, V, D), dtype=torch.float32, device=dev)
              if ctx.needs_input_grad[1] and gyf is not None and D else None)
        if gx is not None or gf is not None:
            _lib.call("dibr_b200_tet_subdivide_backward", dev,
                      B, V, topo.num_edges, D, topo.adj_ptr, topo.adj, topo.adj_edge,
                      None if gx is None else gy.contiguous(), None if gf is None else gyf.contiguous(), gx, gf,
                      what="subdivide_tetmesh")
        return gx, gf, None, None


def subdivide_tetmesh(vertices, tetrahedrons, features=None):
    r"""kaolin.ops.mesh.subdivide_tetmesh: each tetrahedron split into eight at its edge midpoints.

    ``vertices`` (B, V, 3) float32 and the unbatched ``tetrahedrons`` (T, 4) int64 -> (vertices
    (B, V + E, 3), tetrahedrons (8T, 4) int64), and the features (B, V + E, D) when ``features``
    (B, V, D) float32 is given.  Edge e (the grid's unique edges in lexicographic order) becomes vertex
    V + e, at the mean of its endpoints' positions and features; the eight child blocks follow the
    reference's order.  Autograd flows to the vertices and the features, with no atomics.  The topology
    is built on every call, as the reference does.

    Deliberate deviations: only float32 vertices and features and int64 tetrahedrons are accepted; a
    tet index outside [0, V) raises ``IndexError``.
    """
    func = "subdivide_tetmesh"
    typed = [("vertices", vertices, torch.float32), ("tetrahedrons", tetrahedrons, torch.int64)]
    if features is not None:
        typed.append(("features", features, torch.float32))
    _check(func, typed)
    if vertices.dim() != 3 or vertices.shape[-1] != 3:
        raise RuntimeError(f"{func}: expected vertices of shape (B, V, 3), got {list(vertices.shape)}")
    B, V = vertices.shape[:2]
    if features is not None and (features.dim() != 3 or tuple(features.shape[:2]) != (B, V)):
        raise RuntimeError(f"{func}: expected features of shape ({B}, {V}, D), got {list(features.shape)}")
    topo = _TetTopology(func, V, tetrahedrons)
    new_tets = torch.empty((8 * topo.num_tets, 4), dtype=torch.int64, device=vertices.device)
    f = vertices.new_empty((B, V, 0)) if features is None else features.contiguous()
    y, yf = _TetSubdivide.apply(vertices.contiguous(), f, topo, new_tets)
    return (y, new_tets) if features is None else (y, new_tets, yf)
