"""kaolin.metrics.trianglemesh.uniform_laplacian_smoothing on sm_90a kernels, without the V x V matrix
the reference builds (trianglemesh.py:318-350), and point_to_mesh_distance (trianglemesh.py:20-149), every
view in one launch of each kernel (csrc/point_mesh_distance.cu)."""
import torch

from .. import _lib
from ..ops.mesh import _Topology, _apply, _check

__all__ = ["uniform_laplacian_smoothing", "point_to_mesh_distance"]

_DTYPES = {torch.float32: _lib.DTYPE_F32, torch.float64: _lib.DTYPE_F64}
_SCALAR_NAMES = {torch.float16: "Half", torch.bfloat16: "BFloat16", torch.float32: "Float", torch.float64: "Double",
                 torch.uint8: "Byte", torch.int8: "Char", torch.int16: "Short", torch.int32: "Int",
                 torch.int64: "Long", torch.bool: "Bool", torch.complex64: "ComplexFloat",
                 torch.complex128: "ComplexDouble"}


def _dtype_flag(func, dtype):
    """The library's dtype flag, or the reference's AT_DISPATCH_FLOATING_TYPES error."""
    if dtype not in _DTYPES:
        raise RuntimeError(f"\"{func}\" not implemented for '{_SCALAR_NAMES.get(dtype, str(dtype))}'")
    return _DTYPES[dtype]


def _pmd_forward(points, face_vertices, dist, face_idx, dist_type):
    """The library's forward for contiguous points (B, N, 3) and face_vertices (B, F, 3, 3), into the given
    outputs (B, N)."""
    func = "unbatched_triangle_distance_forward_cuda"
    dtype = _dtype_flag(func, points.dtype)
    B, N, F = points.shape[0], points.shape[1], face_vertices.shape[1]
    fwd, _ = _lib.point_mesh_distance_workspace_bytes(B, N, F, dtype, func)
    ws = _lib.scratch(fwd, points.device)
    _lib.call("dibr_b200_point_mesh_distance_forward", points.device, B, N, F, dtype, points, face_vertices, dist,
              face_idx, dist_type, ws, ws.numel(), what=func)


def _pmd_backward(grad_dist, points, face_vertices, face_idx, dist_type, grad_points, grad_face_vertices):
    """The library's backward: grad_points (B, N, 3) written, grad_face_vertices (B, F, 3, 3) added to;
    either may be None."""
    func = "unbatched_triangle_distance_backward_cuda"
    dtype = _dtype_flag(func, points.dtype)
    B, N, F = points.shape[0], points.shape[1], face_vertices.shape[1]
    _, bwd = _lib.point_mesh_distance_workspace_bytes(B, N, F, dtype, func)
    ws = _lib.scratch(bwd, points.device)
    _lib.call("dibr_b200_point_mesh_distance_backward", points.device, B, N, F, dtype, grad_dist, points,
              face_vertices, face_idx, dist_type, grad_points, grad_face_vertices, ws, ws.numel(), what=func)


class _PointToMeshDistance(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pointclouds, face_vertices):
        points, fv = pointclouds.contiguous(), face_vertices.contiguous()
        B, N = points.shape[0], points.shape[1]
        dist = torch.empty((B, N), dtype=points.dtype, device=points.device)
        face_idx = torch.empty((B, N), dtype=torch.long, device=points.device)
        dist_type = torch.empty((B, N), dtype=torch.int32, device=points.device)
        _pmd_forward(points, fv, dist, face_idx, dist_type)
        ctx.save_for_backward(points, fv, face_idx, dist_type)
        ctx.mark_non_differentiable(face_idx, dist_type)
        return dist, face_idx, dist_type

    @staticmethod
    def backward(ctx, grad_dist, grad_face_idx, grad_dist_type):
        points, fv, face_idx, dist_type = ctx.saved_tensors
        grad_points = torch.zeros_like(points) if ctx.needs_input_grad[0] else None
        grad_fv = torch.zeros_like(fv) if ctx.needs_input_grad[1] else None
        if grad_points is not None or grad_fv is not None:
            _pmd_backward(grad_dist.contiguous(), points, fv, face_idx, dist_type, grad_points, grad_fv)
        return grad_points, grad_fv


def point_to_mesh_distance(pointclouds, face_vertices):
    r"""kaolin.metrics.trianglemesh.point_to_mesh_distance: for each point, the squared distance to the
    nearest triangle of its view's mesh, that triangle's index and the distance type.

    ``pointclouds`` (B, N, 3) and ``face_vertices`` (B, F, 3, 3), float32 or float64 CUDA tensors of one
    type -> ``(dist, face_idx, dist_type)``: (B, N) of the input type, int64 and int32.  Distance types:
    0 the face, 1-3 the vertices 0-2, 4 the edge 0-1, 5 the edge 1-2, 6 the edge 2-0.  Autograd flows
    to both inputs.  Every (point, face) pair is evaluated with the reference kernel's arithmetic, so
    outputs and ``grad_points`` equal the reference's CUDA operator bit for bit; the smallest distance
    wins, and among equal distances the lowest face index.  ``dist`` is rounded to float in float64 too,
    as the reference's double kernel does.  All views run in one launch of each kernel, with no host
    read.  Non-contiguous inputs are copied once.

    Deliberate deviations from the reference:

    * NaN faces: a face whose distance is NaN is never chosen unless every face is NaN for the point;
      then the result is NaN, face 0 and face 0's type, as in the reference.  The reference differs when
      a NaN face sits at an index that is a multiple of 512: it then discards the other faces of that
      512-face tile (at index 0, the point's result is NaN).
    * F = 0 raises ``ValueError`` (the reference returns distance 0, face 0, type 0).
    * B = 0 returns (0, N) tensors and N = 0 returns (B, 0) tensors (the reference's ``torch.stack`` of
      an empty list raises for B = 0).
    * ``grad_face_vertices`` is summed in ascending point order, without float atomics, so reruns are
      identical.  It equals the reference bit for bit wherever a face receives at most one point, and
      otherwise differs only by the order of the additions.
    * There is no CPU path.
    """
    func = "point_to_mesh_distance"
    for name, t in (("pointclouds", pointclouds), ("face_vertices", face_vertices)):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{func}: {name} must be a torch.Tensor, got {type(t).__name__}")
        if not t.is_cuda:
            raise RuntimeError(f"{func}: {name} must be a CUDA tensor (kaolin_b200 has no CPU path)")
    if pointclouds.device != face_vertices.device:
        raise RuntimeError(f"{func}: expected both tensors on one device, got {pointclouds.device} and "
                           f"{face_vertices.device}")
    if pointclouds.dim() != 3 or pointclouds.shape[2] != 3:
        raise ValueError(f"{func}: expected pointclouds of shape (B, N, 3), got {tuple(pointclouds.shape)}")
    if face_vertices.dim() != 4 or tuple(face_vertices.shape[2:]) != (3, 3):
        raise ValueError(f"{func}: expected face_vertices of shape (B, F, 3, 3), got {tuple(face_vertices.shape)}")
    if pointclouds.shape[0] != face_vertices.shape[0]:
        raise ValueError(f"{func}: expected pointclouds and face_vertices of one batch size, got "
                         f"{pointclouds.shape[0]} and {face_vertices.shape[0]}")
    _dtype_flag("unbatched_triangle_distance_forward_cuda", pointclouds.dtype)
    if face_vertices.dtype != pointclouds.dtype:
        raise RuntimeError(f"{func}: expected face_vertices of type {pointclouds.dtype}, got {face_vertices.dtype}")
    if face_vertices.shape[1] == 0:
        raise ValueError(f"{func}: the meshes have no face (F = 0)")
    return _PointToMeshDistance.apply(pointclouds, face_vertices)


def uniform_laplacian_smoothing(vertices, faces):
    r"""Each vertex moved to the mean of its neighbours: ``(L + I) @ vertices`` for the uniform
    Laplacian L of ``faces``; vertices (B, V, 3) float32 -> (B, V, 3), with autograd to vertices.
    A vertex without neighbours goes to 0, as in the reference."""
    func = "uniform_laplacian_smoothing"
    _check(func, [("vertices", vertices, torch.float32), ("faces", faces, torch.int64)])
    topo = _Topology(func, vertices.shape[1], faces)
    return _apply(func, topo, vertices, True)
