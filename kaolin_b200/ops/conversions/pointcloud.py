"""kaolin.ops.conversions.pointclouds_to_voxelgrids on sm_90a kernels (csrc/voxelize.cu), and the
voxelization both conversions into voxel grids share.

The reference (pointcloud.py:22-141) quantises every point, runs ``torch.unique`` over all of them,
builds a sparse tensor and densifies it.  Here one kernel sets one bit per point in a bit grid of
B res^3 bits, and one streaming kernel expands the bits into the dense grid; the sparse result is
emitted from the bits in grid order, which is the reference's sorted order.
"""
import torch

from ... import _lib

__all__ = ["pointclouds_to_voxelgrids"]

MAX_DEPTH = 24   # DIBR_B200_VOXELIZE_MAX_DEPTH: levels of subdivision below a face


def _check_resolution(func, resolution, least):
    if not isinstance(resolution, int):
        raise TypeError(f"Expected resolution to be int but got {type(resolution)}.")
    if resolution < least:
        raise ValueError(f"{func}: resolution must be at least {least}, got {resolution}")


def _check_points(func, name, points):
    if not isinstance(points, torch.Tensor):
        raise TypeError(f"{func}: expected {name} to be a torch.Tensor, got {type(points)}")
    if not points.is_cuda:
        raise NotImplementedError(f"{func} does not support CPU.")
    if points.dim() != 3 or points.shape[2] != 3:
        raise ValueError(f"{func}: expected {name} of shape (batch_size, num_points, 3), got {list(points.shape)}")


def _normalize(points, origin, scale):
    """The reference's normalisation, as its torch expression, so that promotion and rounding match."""
    if origin is None:
        origin = torch.min(points, dim=1)[0]
    if scale is None:
        scale = torch.max(torch.max(points, dim=1)[0] - origin, dim=1)[0]
    return (points - origin.unsqueeze(1)) / scale.view(-1, 1, 1)


def _voxelize(func, points, faces, resolution, return_sparse):
    """Normalised points (B, P, 3) float32 / float64 and faces (F, 3) int64 or None -> the grid, dense
    or sparse.  Host reads: one when there are faces (the status) or when sparse (the status and the
    number of set voxels, together), none otherwise."""
    if points.dtype not in (torch.float32, torch.float64):
        raise TypeError(f"{func}: normalized points must be float32 or float64, got {points.dtype}")
    B, P = points.shape[0], points.shape[1]
    F = 0 if faces is None else faces.shape[0]
    dev, dtype, res = points.device, points.dtype, resolution
    size = (B, res, res, res)
    if B == 0:
        if return_sparse:
            return torch.sparse_coo_tensor(torch.zeros((4, 0), dtype=torch.int64, device=dev),
                                           torch.zeros(0, dtype=dtype, device=dev), size)
        return torch.zeros(size, dtype=dtype, device=dev)
    flag = _lib.DTYPE_F32 if dtype == torch.float32 else _lib.DTYPE_F64
    nbytes = _lib.voxelize_workspace_bytes(B, F, res, func)
    ws = _lib.scratch(nbytes, dev)
    info = torch.empty(4, dtype=torch.int64, device=dev)
    points = points.contiguous()
    _lib.call("dibr_b200_voxelize_mark", dev, B, P, F, res, flag, points, faces if F else None, int(bool(return_sparse)),
              info, ws, nbytes, what=func)
    out = None
    if not return_sparse:
        out = torch.empty(size, dtype=dtype, device=dev)
        _lib.call("dibr_b200_voxelize_dense", dev, B, F, res, flag, out, ws, nbytes, what=func)
    if F == 0 and not return_sparse:
        return out
    flags, bad_face, deep_face, nnz = info.tolist()          # the call's one device-to-host read
    if flags & 1:
        raise IndexError(f"{func}: face {bad_face % F} (view {bad_face // F}) indexes a vertex outside "
                         f"[0, {P})")
    if flags & 2:
        raise ValueError(f"{func}: face {deep_face % F} (view {deep_face // F}) needs more than "
                         f"{MAX_DEPTH} levels of subdivision at resolution {res}")
    if not return_sparse:
        return out
    if nnz > 2 ** 31 - 1:
        raise ValueError(f"{func}: {nnz} occupied voxels exceed the sparse result's limit of 2^31 - 1")
    indices = torch.empty((4, nnz), dtype=torch.int64, device=dev)
    _lib.call("dibr_b200_voxelize_sparse", dev, B, F, res, nnz, indices, ws, nbytes, what=func)
    return torch.sparse_coo_tensor(indices, torch.ones(nnz, dtype=dtype, device=dev), size, check_invariants=False)



def pointclouds_to_voxelgrids(pointclouds, resolution, origin=None, scale=None, return_sparse=False):
    r"""kaolin.ops.conversions.pointclouds_to_voxelgrids: the occupancy grid of each point cloud.

    Points are normalised as ``(pointclouds - origin) / scale`` (the reference's code divides; its
    docstring says multiplies), ``origin`` (B, 3) defaulting to the per-view minimum and ``scale``
    (B,) to the largest extent, computed with the reference's torch expression, so the grid's dtype
    follows torch's type promotion.  A point sets voxel ``round(p * (resolution - 1))`` (half to
    even) when all three indices lie in ``[0, resolution - 1]``; a NaN coordinate drops the point,
    as in the reference on the CPU and on CUDA.

    Returns a (B, resolution, resolution, resolution) tensor of 0 and 1 in the normalised points'
    dtype, equal to the reference bit for bit; with ``return_sparse`` a ``sparse_coo`` tensor of the
    same size, its indices in sorted (view, x, y, z) order, values ones, not marked coalesced.  All
    views go through one launch per kernel; the dense result needs no host read, the sparse one
    reads its size back once.

    Deliberate deviations from the reference:

    - ``resolution < 1`` raises ValueError;
    - a batch of 0 views returns an empty grid;
    - only float32 and float64 normalised points are accepted (TypeError otherwise), and there is no
      CPU path (a CPU tensor raises NotImplementedError).
    """
    func = "pointclouds_to_voxelgrids"
    _check_resolution(func, resolution, 1)
    _check_points(func, "pointclouds", pointclouds)
    points = _normalize(pointclouds, origin, scale)
    return _voxelize(func, points, None, resolution, return_sparse)
