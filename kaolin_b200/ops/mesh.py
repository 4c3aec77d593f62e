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

``check_sign`` (check_sign.py) labels points inside or outside a watertight mesh, equal to the
reference's CUDA operator bit for bit, with its faces binned on a y-z grid instead of tested against
every point (csrc/check_sign.cu); ``CheckSign`` builds the mesh once for many point sets::

    S = CheckSign(verts, faces)               # Simplicits, occupancy sampling: many point sets, one mesh
    inside = S(points)                        # (B, N) bool, no host synchronisation

``sample_points``, ``packed_sample_points``, ``face_areas`` and ``packed_face_areas``
(trianglemesh.py:30-311) sample a surface by area with a stated Philox random stream and a float64 CDF
per view (csrc/sample_points.cu); ``SurfaceSampler`` keeps the topology its backward needs and never
reads the host::

    S = SurfaceSampler(V, faces)              # DMTet: fixed topology, sampled every step
    points, face_choices = S(vertices, 50000)
"""
import torch

from .. import _lib
from ..render.mesh import _host

__all__ = ["adjacency_matrix", "uniform_laplacian", "compute_vertex_normals", "average_face_vertex_features",
           "UniformLaplacian", "subdivide_trianglemesh", "LoopSubdivision", "subdivide_tetmesh", "check_sign",
           "CheckSign", "face_areas", "packed_face_areas", "sample_points", "packed_sample_points",
           "SurfaceSampler"]


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
        ws = _lib.scratch(nbytes, dev)
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


_CHECK_SIGN_DTYPES = {torch.float32: _lib.DTYPE_F32, torch.float64: _lib.DTYPE_F64}


def _check_sign_args(verts, faces, points, hash_resolution):
    """check_sign.py:104-136, in its order, with its types and messages (``points`` None: CheckSign)."""
    if points is not None:
        assert verts.device == points.device
        assert faces.device == points.device
    else:
        assert faces.device == verts.device
    if not faces.dtype == torch.int64:
        raise TypeError(f"Expected faces entries to be torch.int64 "
                        f"but got {faces.dtype}.")
    if not isinstance(hash_resolution, int):
        raise TypeError(f"Expected hash_resolution to be int "
                        f"but got {type(hash_resolution)}.")
    if verts.ndim != 3:
        raise ValueError(f"Expected verts to have 3 dimensions "
                         f"but got {verts.ndim} dimensions.")
    if faces.ndim != 2:
        raise ValueError(f"Expected faces to have 2 dimensions "
                         f"but got {faces.ndim} dimensions.")
    if points is not None and points.ndim != 3:
        raise ValueError(f"Expected points to have 3 dimensions "
                         f"but got {points.ndim} dimensions.")
    if verts.shape[2] != 3:
        raise ValueError(f"Expected verts to have 3 coordinates "
                         f"but got {verts.shape[2]} coordinates.")
    if faces.shape[1] != 3:
        raise ValueError(f"Expected faces to have 3 vertices "
                         f"but got {faces.shape[1]} vertices.")
    if points is not None and points.shape[2] != 3:
        raise ValueError(f"Expected points to have 3 coordinates "
                         f"but got {points.shape[2]} coordinates.")


def _check_sign_dtype(func, dtype, named):
    """CUDA tensors of one type, float32 or float64: the reference's operator takes verts and points of
    one type (at::checkAllSameType)."""
    _host.check_tensors(func, named, dtype=None)
    if dtype not in _CHECK_SIGN_DTYPES:
        raise RuntimeError(f"\"{func}\" not implemented for '{str(dtype).replace('torch.', '')}' "
                           "(kaolin_b200 takes verts and points as float32 or float64)")
    for name, t in named:
        if t.dtype != dtype:
            raise RuntimeError(f"{func}: expected {name} of type {dtype}, got {t.dtype}")


class CheckSign:
    r"""The point-in-mesh test of one (batched) mesh, built once.

    ``S = CheckSign(verts, faces)`` normalises the mesh and bins its faces; ``S(points)`` then returns
    ``check_sign(verts, faces, points)`` without a host synchronisation, for labelling many point sets
    against one mesh (uniform samples in its box, occupancy and SDF pre-training)::

        S = CheckSign(verts, faces)               # one device-to-host read: the face-index check
        inside = S(points)                        # (B, N) bool, as check_sign(verts, faces, points)

    ``verts`` (B, V, 3) float32 or float64 and ``faces`` (F, 3) int64 on one CUDA device; the points
    must have the verts' type and batch size.  The reference normalises by each mesh's extent on every
    call; the mesh is fixed here at build, so the result is the same.  Later changes to ``verts`` do not
    reach ``S``.  The argument errors are ``check_sign``'s; a face index outside [0, V) raises
    ``IndexError``.
    """

    def __init__(self, verts, faces):
        func = "CheckSign"
        _check_sign_args(verts, faces, None, 0)
        _check_sign_dtype(func, verts.dtype, [("verts", verts)])
        _check(func, [("faces", faces, torch.int64)])
        self.dtype, self.device = verts.dtype, verts.device
        B, V, _ = verts.shape
        F = faces.shape[0]
        self.batch_size, self.num_vertices, self.num_faces = B, V, F
        if B == 0:
            return
        dtype = _CHECK_SIGN_DTYPES[verts.dtype]
        nbytes, _ = _lib.check_sign_workspace_bytes(B, F, 0, dtype, func)
        self._mesh = _lib.scratch(nbytes, verts.device)
        status = torch.empty(1, dtype=torch.int32, device=verts.device)
        _lib.call("dibr_b200_check_sign_build", verts.device, B, V, F, dtype, verts.contiguous(),
                  faces.contiguous(), status, self._mesh, self._mesh.numel(), what=func)
        if status.item():                                 # the build's one device-to-host read
            raise IndexError(f"{func}: faces holds an index outside [0, {V})")

    def __call__(self, points):
        func = "CheckSign"
        if points.ndim != 3 or points.shape[2] != 3:
            raise ValueError(f"{func}: expected points of shape (B, N, 3), got {list(points.shape)}")
        _check_sign_dtype(func, self.dtype, [("points", points)])
        if points.device != self.device:
            raise RuntimeError(f"{func}: expected points on {self.device}, got {points.device}")
        B, N = self.batch_size, points.shape[1]
        if points.shape[0] != B:
            raise ValueError(f"{func}: expected points of batch size {B}, got {points.shape[0]}")
        out = torch.empty((B, N), dtype=torch.bool, device=points.device)
        if B == 0 or N == 0:
            return out
        dtype = _CHECK_SIGN_DTYPES[self.dtype]
        _, nbytes = _lib.check_sign_workspace_bytes(B, self.num_faces, N, dtype, func)
        ws = _lib.scratch(nbytes, points.device)
        _lib.call("dibr_b200_check_sign_query", points.device, B, self.num_faces, N, dtype, points.contiguous(),
                  self._mesh, self._mesh.numel(), out, ws, ws.numel(), what=func)
        return out


def check_sign(verts, faces, points, hash_resolution=512):
    r"""kaolin.ops.mesh.check_sign: whether each point lies inside a watertight triangle mesh.

    ``verts`` (B, V, 3), ``faces`` (F, 3) int64 and ``points`` (B, N, 3) -> (B, N) bool.  Per view, the
    vertices and points are divided by the mesh's largest extent over all V vertices, and a ray from
    each point along +x is tested against every face; a point is inside when it crosses an odd number of
    faces.  Equal to the reference's CUDA operator bit for bit in float32 and float64: every comparison
    follows its compiled arithmetic, including the edge and vertex tie-breaking.  The faces are binned
    on a y-z grid, so each point is tested against its cell's faces only.  The mesh is built on every
    call, as the reference does (one device-to-host read, the face-index check); ``CheckSign`` builds it
    once.  ``hash_resolution`` is type-checked as in the reference and otherwise unused (the reference
    uses it on its CPU path only).  The argument errors are the reference's, in its order.

    Deliberate deviations: ``verts`` and ``points`` must be float32 or float64 CUDA tensors of one type
    and one batch size (there is no CPU path); F = 0 gives all ``False`` (the reference's launch fails);
    B = 0 gives a (0, N) tensor (the reference's ``torch.stack([])`` raises); a face index outside
    [0, V) raises ``IndexError`` (the reference's ``index_select`` faults on the device).
    """
    _check_sign_args(verts, faces, points, hash_resolution)
    _check_sign_dtype("check_sign", verts.dtype, [("verts", verts), ("points", points)])
    if verts.shape[0] != points.shape[0]:
        raise ValueError(f"check_sign: expected verts and points of one batch size, "
                         f"got {verts.shape[0]} and {points.shape[0]}")
    return CheckSign(verts, faces)(points)


# ---------------------------------------------------------------------------------------------
# Face areas and surface sampling (csrc/sample_points.cu).

_SAMPLE_DTYPES = {torch.float32: _lib.DTYPE_F32, torch.float64: _lib.DTYPE_F64}
_BAD_INDEX, _BAD_DISTRIBUTION = 1, 2          # DIBR_B200_SAMPLE_* status bits


def _sample_dtype(func, named):
    """float32 or float64, one type for every named tensor (None skipped)."""
    named = [(n, t) for n, t in named if t is not None]
    for name, t in named:
        if t.dtype not in _SAMPLE_DTYPES:
            raise TypeError(f"{func}: expected {name} of type float32 or float64, got {t.dtype}")
        if t.dtype != named[0][1].dtype:
            raise TypeError(f"{func}: expected {name} of type {named[0][1].dtype}, got {t.dtype}")


def _triangles(func, faces):
    if not isinstance(faces, torch.Tensor) or faces.dim() != 2:
        raise ValueError(f"{func}: expected faces of shape (num_faces, 3)")
    if faces.shape[-1] != 3:
        raise NotImplementedError(f"{func} is only implemented for triangle meshes")
    if faces.dtype != torch.int64:
        raise TypeError(f"{func}: expected faces of type torch.int64, got {faces.dtype}")


class _Views:
    """The views of one call (include/dibr_b200.h): view b owns faces [face_off[b], face_off[b + 1]) of
    ``faces``, row g - b * fstride, vertex b * vstride + index, every index in [0, num_vertices)."""

    def __init__(self, batch, faces, num_vertices, fstride, vstride, face_off):
        self.batch, self.faces, self.face_off = batch, faces, face_off
        self.dims = (batch, batch * fstride if fstride else faces.shape[0], num_vertices, fstride, vstride)

    @staticmethod
    def dense(vertices, faces):
        B, V = vertices.shape[:2]
        F = faces.shape[0]
        off = torch.arange(B + 1, dtype=torch.int64, device=faces.device) * F
        return _Views(B, faces, V, F, V, off)

    @staticmethod
    def packed(func, vertices, first_idx_vertices, faces, num_faces_per_mesh):
        """The merged faces (faces + each mesh's first vertex) and their views, without a host read."""
        dev = vertices.device
        B, F = num_faces_per_mesh.shape[0], faces.shape[0]
        counts = num_faces_per_mesh.reshape(-1).to(device=dev, dtype=torch.int64)
        if not num_faces_per_mesh.is_cuda and int(num_faces_per_mesh.sum()) != F:
            raise ValueError(f"{func}: num_faces_per_mesh sums to {int(num_faces_per_mesh.sum())}, "
                             f"but faces has {F} rows")
        # face_off is clamped to [0, F] and ends at F, so that inconsistent counts on the device give
        # wrong views but never an access outside the faces
        off = torch.zeros(B + 1, dtype=torch.int64, device=dev)
        off[1:] = torch.cumsum(counts.clamp(min=0), 0).clamp(max=F)
        off[B] = F
        first = first_idx_vertices[:B].reshape(-1).to(device=dev, dtype=torch.int64)
        merged = faces + torch.repeat_interleave(first, counts.clamp(min=0), output_size=F)[:, None]
        return _Views(B, merged.contiguous(), vertices.shape[0], 0, 0, off)


def _call_face_areas(func, vertices, views, status):
    areas = vertices.new_empty(views.dims[1])
    _lib.call("dibr_b200_face_areas_forward", vertices.device, *views.dims, _SAMPLE_DTYPES[vertices.dtype],
              views.face_off, views.faces, vertices, areas, status, what=func)
    return areas


class _FaceAreas(torch.autograd.Function):
    @staticmethod
    def forward(ctx, vertices, views, topo, status):
        ctx.save_for_backward(vertices)
        ctx.views, ctx.topo = views, topo
        return _call_face_areas("face_areas", vertices, views, status)

    @staticmethod
    def backward(ctx, grad):
        vertices, = ctx.saved_tensors
        views, topo = ctx.views, ctx.topo
        dtype = _SAMPLE_DTYPES[vertices.dtype]
        _, nbytes = _lib.sample_points_workspace_bytes(views.batch, views.dims[1], 0, dtype, "face_areas")
        ws = _lib.scratch(nbytes, vertices.device)
        gv = torch.empty_like(vertices)
        _lib.call("dibr_b200_face_areas_backward", vertices.device, *views.dims, dtype, views.face_off,
                  views.faces, vertices, grad.contiguous(), topo.corner_ptr, topo.corners, gv, ws, ws.numel(),
                  what="face_areas")
        return gv, None, None, None


def _wants_grad(*tensors):
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


def _status_errors(func, status, topo):
    """The functional forms' one device-to-host read: the topology build's status words (when a
    topology was built) and the sampling status word."""
    edges, topo_error, flags = status.tolist()
    if topo is not None:
        topo._finish(func, edges, topo_error)
    if flags & _BAD_INDEX:
        raise IndexError(f"{func}: faces holds an index outside the vertices")
    if flags & _BAD_DISTRIBUTION:
        raise ValueError(f"{func}: the face areas are not a distribution (a negative, NaN or infinite area, "
                         "or a zero total)")


def _face_areas(func, vertices, views, num_vertices, topo_faces):
    if views.dims[1] == 0:
        return vertices.new_zeros(0)
    status = torch.zeros(3, dtype=torch.int32, device=vertices.device)
    topo = _Topology(func, num_vertices, topo_faces, status=status) if _wants_grad(vertices) else None
    areas = _FaceAreas.apply(vertices.contiguous(), views, topo, status[2:])
    _status_errors(func, status, topo)
    return areas


def face_areas(vertices, faces):
    r"""kaolin.ops.mesh.face_areas: the area of every face, (B, F) of ``vertices``' type, with autograd
    to ``vertices`` (B, V, 3) float32 or float64; ``faces`` (F, 3) int64.  The reference's rounding,
    bit for bit; a zero-area face's gradient is NaN, as the reference's autograd gives.  One
    device-to-host read per call.  Deliberate deviations: a face index outside [0, V) raises
    ``IndexError``; other float types raise ``TypeError``."""
    func = "face_areas"
    _triangles(func, faces)
    _sample_dtype(func, [("vertices", vertices)])
    _host.check_tensors(func, [("vertices", vertices), ("faces", faces)], dtype=None)
    if vertices.dim() != 3 or vertices.shape[-1] != 3:
        raise ValueError(f"{func}: expected vertices of shape (B, V, 3), got {list(vertices.shape)}")
    B, F = vertices.shape[0], faces.shape[0]
    if B == 0:
        return vertices.new_zeros((0, F))
    faces = faces.contiguous()
    return _face_areas(func, vertices, _Views.dense(vertices, faces), vertices.shape[1], faces).view(B, F)


def packed_face_areas(vertices, first_idx_vertices, faces, num_faces_per_mesh):
    r"""kaolin.ops.mesh.packed_face_areas: the area of every packed face, (sum F,), with autograd to the
    packed ``vertices`` (sum V, 3).  ``first_idx_vertices`` (B + 1) and ``num_faces_per_mesh`` (B)
    may live on the CPU or the GPU.  As ``face_areas``, on the merged faces."""
    func = "packed_face_areas"
    _triangles(func, faces)
    _sample_dtype(func, [("vertices", vertices)])
    _host.check_tensors(func, [("vertices", vertices), ("faces", faces)], dtype=None)
    if vertices.dim() != 2 or vertices.shape[-1] != 3:
        raise ValueError(f"{func}: expected vertices of shape (num_vertices, 3), got {list(vertices.shape)}")
    if num_faces_per_mesh.shape[0] == 0:
        return vertices.new_zeros(faces.shape[0])
    views = _Views.packed(func, vertices, first_idx_vertices, faces, num_faces_per_mesh)
    return _face_areas(func, vertices, views, vertices.shape[0], views.faces)


class _SamplePoints(torch.autograd.Function):
    """vertices, face_features (B*F, 3, D) or an empty placeholder -> points, face_choices, features
    (an empty (B, N, 0) without face_features)."""

    @staticmethod
    def forward(ctx, vertices, face_features, views, num_samples, areas, key, topo, status):
        dev = vertices.device
        B, nf = views.batch, views.dims[1]
        D = face_features.shape[-1] if face_features.dim() == 4 else 0
        dtype = _SAMPLE_DTYPES[vertices.dtype]
        fwd, _ = _lib.sample_points_workspace_bytes(B, nf, num_samples, dtype, "sample_points")
        ws = _lib.scratch(fwd, dev)
        points = vertices.new_empty((B, num_samples, 3))
        choices = torch.empty((B, num_samples), dtype=torch.int64, device=dev)
        features = vertices.new_empty((B, num_samples, D))
        _lib.call("dibr_b200_sample_points_forward", dev, *views.dims, dtype, num_samples, D, views.face_off,
                  views.faces, vertices, areas, face_features if D else None, key, points, choices,
                  features if D else None, status, ws, ws.numel(), what="sample_points")
        ctx.mark_non_differentiable(choices)
        ctx.save_for_backward(choices, key)
        ctx.views, ctx.topo, ctx.num_samples, ctx.D = views, topo, num_samples, D
        ctx.shapes = (vertices.shape, face_features.shape)
        return points, choices, features

    @staticmethod
    def backward(ctx, grad_points, _grad_choices, grad_features):
        choices, key = ctx.saved_tensors
        views, topo, N, D = ctx.views, ctx.topo, ctx.num_samples, ctx.D
        dev = choices.device
        dtype_t = grad_points.dtype
        gv = torch.empty(ctx.shapes[0], dtype=dtype_t, device=dev) if ctx.needs_input_grad[0] else None
        gf = torch.empty(ctx.shapes[1], dtype=dtype_t, device=dev) if ctx.needs_input_grad[1] and D else None
        if gv is None and gf is None:
            return None, None, None, None, None, None, None, None
        dtype = _SAMPLE_DTYPES[dtype_t]
        _, nbytes = _lib.sample_points_workspace_bytes(views.batch, views.dims[1], N, dtype, "sample_points")
        ws = _lib.scratch(nbytes, dev)
        _lib.call("dibr_b200_sample_points_backward", dev, *views.dims, dtype, N, D, views.face_off, key, choices,
                  grad_points.contiguous() if gv is not None else None,
                  grad_features.contiguous() if gf is not None else None,
                  topo.corner_ptr if gv is not None else None, topo.corners if gv is not None else None, gv, gf,
                  ws, ws.numel(), what="sample_points")
        return gv, gf, None, None, None, None, None, None


def _draw_key(device):
    """One 64-bit Philox key drawn on the device from torch's CUDA generator: ``torch.manual_seed``
    makes a call reproducible, and nothing is read back to the host."""
    return torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64, device=device)


def _sample_args(func, vertices, views, num_samples, areas, areas_shape, face_features):
    """Checks of the sampling arguments; -> (num_samples, areas as float64 or None, face_features)."""
    if isinstance(num_samples, bool) or not isinstance(num_samples, int) or num_samples < 0:
        raise ValueError(f"{func}: num_samples must be an int >= 0, got {num_samples!r}")
    _sample_dtype(func, [("vertices", vertices), ("face_features", face_features)])
    if areas is not None:
        _sample_dtype(func, [("areas", areas)])
        if tuple(areas.shape) != tuple(areas_shape):
            raise ValueError(f"{func}: expected areas of shape {list(areas_shape)}, got {list(areas.shape)}")
        areas = areas.detach().to(torch.float64).contiguous()
    if face_features is not None:
        B, F = views.batch, views.dims[3]
        if face_features.dim() != 4 or tuple(face_features.shape[:3]) != (B, F, 3):
            raise ValueError(f"{func}: expected face_features of shape ({B}, {F}, 3, D), "
                             f"got {list(face_features.shape)}")
        face_features = face_features.contiguous()
    return num_samples, areas, face_features


def _run_sample(vertices, views, num_samples, areas, face_features, key, topo, status):
    ff = face_features if face_features is not None else vertices.new_empty(0)
    points, choices, features = _SamplePoints.apply(vertices.contiguous(), ff, views, num_samples, areas, key, topo,
                                                    status)
    return (points, choices) if face_features is None else (points, choices, features)


def _empty_samples(vertices, B, num_samples, face_features):
    out = (vertices.new_zeros((B, num_samples, 3)),
           torch.zeros((B, num_samples), dtype=torch.int64, device=vertices.device))
    if face_features is not None:
        out += (vertices.new_zeros((B, num_samples, face_features.shape[-1])),)
    return out


def _sample_points(vertices, faces, num_samples, areas, face_features, key):
    """``sample_points`` with the Philox key given (a (1,) int64 CUDA tensor)."""
    func = "sample_points"
    _triangles(func, faces)
    _host.check_tensors(func, [("vertices", vertices), ("faces", faces)], dtype=None)
    if vertices.dim() != 3 or vertices.shape[-1] != 3:
        raise ValueError(f"{func}: expected vertices of shape (B, V, 3), got {list(vertices.shape)}")
    B, F = vertices.shape[0], faces.shape[0]
    for name, t in (("areas", areas), ("face_features", face_features)):
        if t is not None:
            _host.check_tensors(func, [("vertices", vertices), (name, t)], dtype=None)
    if F == 0:
        raise ValueError(f"{func}: cannot sample a mesh without faces")
    if B == 0:
        _sample_args(func, vertices, _Views(0, faces, 0, F, 0, None), num_samples, areas, (0, F), face_features)
        return _empty_samples(vertices, 0, num_samples, face_features)
    faces = faces.contiguous()
    views = _Views.dense(vertices, faces)
    num_samples, areas, face_features = _sample_args(func, vertices, views, num_samples, areas, (B, F), face_features)
    status = torch.zeros(3, dtype=torch.int32, device=vertices.device)
    topo = _Topology(func, vertices.shape[1], faces, status=status) if _wants_grad(vertices) else None
    out = _run_sample(vertices, views, num_samples, areas, face_features, key, topo, status[2:])
    _status_errors(func, status, topo)
    return out


def sample_points(vertices, faces, num_samples, areas=None, face_features=None):
    r"""kaolin.ops.mesh.sample_points: ``num_samples`` points per view, uniformly over the surface.

    ``vertices`` (B, V, 3) float32 or float64, ``faces`` (F, 3) int64 -> (points (B, N, 3), face_choices
    (B, N) int64), and the interpolated features (B, N, D) when ``face_features`` (B, F, 3, D) of the
    vertices' type is given.  Autograd flows to ``vertices`` and ``face_features``; ``areas`` (B, F),
    the unnormalised distribution of the faces, gets none, as in the reference.

    Each face is chosen with probability proportional to its area and each point placed with the
    reference's barycentric rounding.  The random stream is a stated contract (csrc/sample_points.cu):
    one 64-bit key is drawn on the device from torch's CUDA generator, so ``torch.manual_seed``
    reproduces a call bit for bit.  The backward has no float atomics: it is bit-reproducible.  One
    device-to-host read per call, the status word.  Views of more than 2^24 faces work.

    Deliberate deviations: an invalid distribution (a negative, NaN or infinite area, a zero total,
    NaN vertices) raises ``ValueError`` as the reference's Categorical does, and a face index outside
    [0, V) raises ``IndexError``; F = 0 raises ``ValueError``; B = 0 gives empty outputs; only float32
    and float64 are accepted (``TypeError``), and ``face_features`` must have the vertices' type.
    ``SurfaceSampler`` builds the topology once and makes no host read.
    """
    _host.check_tensors("sample_points", [("vertices", vertices)], dtype=None)
    return _sample_points(vertices, faces, num_samples, areas, face_features, _draw_key(vertices.device))


def _packed_sample_points(vertices, first_idx_vertices, faces, num_faces_per_mesh, num_samples, areas, key):
    """``packed_sample_points`` with the Philox key given."""
    func = "packed_sample_points"
    _triangles(func, faces)
    _host.check_tensors(func, [("vertices", vertices), ("faces", faces)], dtype=None)
    if vertices.dim() != 2 or vertices.shape[-1] != 3:
        raise ValueError(f"{func}: expected vertices of shape (num_vertices, 3), got {list(vertices.shape)}")
    if areas is not None:
        _host.check_tensors(func, [("vertices", vertices), ("areas", areas)], dtype=None)
    B = num_faces_per_mesh.shape[0]
    if faces.shape[0] == 0:
        raise ValueError(f"{func}: cannot sample a mesh without faces")
    if B == 0:
        _sample_args(func, vertices, _Views(0, faces, 0, 0, 0, None), num_samples, areas, (faces.shape[0],), None)
        return _empty_samples(vertices, 0, num_samples, None)
    views = _Views.packed(func, vertices, first_idx_vertices, faces.contiguous(), num_faces_per_mesh)
    num_samples, areas, _ = _sample_args(func, vertices, views, num_samples, areas, (faces.shape[0],), None)
    status = torch.zeros(3, dtype=torch.int32, device=vertices.device)
    topo = _Topology(func, vertices.shape[0], views.faces, status=status) if _wants_grad(vertices) else None
    out = _run_sample(vertices, views, num_samples, areas, None, key, topo, status[2:])
    _status_errors(func, status, topo)
    return out


def packed_sample_points(vertices, first_idx_vertices, faces, num_faces_per_mesh, num_samples, areas=None):
    r"""kaolin.ops.mesh.packed_sample_points: ``sample_points`` on packed meshes.

    ``vertices`` (sum V, 3), ``first_idx_vertices`` (B + 1), ``faces`` (sum F, 3) int64 indexing each
    mesh's own vertices, ``num_faces_per_mesh`` (B) -> (points (B, N, 3), the chosen faces as indices
    of the packed faces (B, N) int64), as the reference returns them; ``areas`` (sum F,) optional.
    Autograd flows to ``vertices``.  The errors and deviations are ``sample_points``'; an empty mesh is
    an invalid distribution."""
    _host.check_tensors("packed_sample_points", [("vertices", vertices)], dtype=None)
    return _packed_sample_points(vertices, first_idx_vertices, faces, num_faces_per_mesh, num_samples, areas,
                                 _draw_key(vertices.device))


class SurfaceSampler:
    r"""``sample_points`` on one fixed topology, built once.

    ``S = SurfaceSampler(num_vertices, faces)`` checks ``faces`` (F, 3) int64 once (one device-to-host
    read) and keeps the corner CSR the backward gathers over; ``S(vertices, num_samples, areas=None,
    face_features=None)`` then returns what ``sample_points`` returns, for any batch size, with no
    device-to-host read in the forward or the backward::

        S = SurfaceSampler(V, faces)                    # DMTet-style loops, deforming a sphere
        points, face_choices = S(vertices, 50000)        # (B, N, 3), (B, N)

    Because a call never reads the host, it cannot raise on its data: a view whose areas are not a
    distribution (a negative, NaN or infinite area, or a zero total, e.g. from NaN vertices) gets face
    index -1, NaN points and NaN features, and contributes zero gradients.
    """

    def __init__(self, num_vertices, faces):
        func = "SurfaceSampler"
        _triangles(func, faces)
        if faces.shape[0] == 0:
            raise ValueError(f"{func}: cannot sample a mesh without faces")
        self._topo = _Topology(func, num_vertices, faces)
        self.num_vertices, self.faces = self._topo.num_vertices, self._topo.faces

    def __call__(self, vertices, num_samples, areas=None, face_features=None):
        func = "SurfaceSampler"
        V, F = self.num_vertices, self.faces.shape[0]
        _host.check_tensors(func, [("vertices", vertices), ("faces", self.faces)], dtype=None)
        for name, t in (("areas", areas), ("face_features", face_features)):
            if t is not None:
                _host.check_tensors(func, [("vertices", vertices), (name, t)], dtype=None)
        if vertices.dim() != 3 or tuple(vertices.shape[1:]) != (V, 3):
            raise ValueError(f"{func}: expected vertices of shape (B, {V}, 3), got {list(vertices.shape)}")
        B = vertices.shape[0]
        if B == 0:
            _sample_args(func, vertices, _Views(0, self.faces, 0, F, 0, None), num_samples, areas, (0, F),
                         face_features)
            return _empty_samples(vertices, 0, num_samples, face_features)
        views = _Views.dense(vertices, self.faces)
        num_samples, areas, face_features = _sample_args(func, vertices, views, num_samples, areas, (B, F),
                                                         face_features)
        status = torch.empty(1, dtype=torch.int32, device=vertices.device)   # written, never read
        return _run_sample(vertices, views, num_samples, areas, face_features, _draw_key(vertices.device), self._topo,
                           status)
