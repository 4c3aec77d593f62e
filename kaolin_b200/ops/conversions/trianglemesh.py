"""kaolin.ops.conversions.trianglemeshes_to_voxelgrids on sm_90a kernels (csrc/voxelize.cu).

The reference (trianglemesh.py:29-110) loops over the views in Python and subdivides each view
level by level (kaolin/ops/mesh/trianglemesh.py:340-458): every level reads a count back to the
host, filters with a boolean mask and runs ``torch.unique`` over every vertex made so far.  Here the
faces of every view are cut into work items in one count pass and a scan, each item walks its part
of a face's subdivision depth first and sets the bits of the midpoints it makes, and the bits become
the grid as in pointclouds_to_voxelgrids.  The call makes one device-to-host read, the status.
"""
import torch

from .pointcloud import _check_points, _check_resolution, _normalize, _voxelize

__all__ = ["trianglemeshes_to_voxelgrids"]


def trianglemeshes_to_voxelgrids(vertices, faces, resolution, origin=None, scale=None, return_sparse=False):
    r"""kaolin.ops.conversions.trianglemeshes_to_voxelgrids: the surface voxel grid of each mesh.

    ``vertices`` (B, V, 3) are normalised as ``(vertices - origin) / scale`` with the reference's
    defaults and torch expression (over every vertex, referenced or not; the grid's dtype follows
    torch's type promotion).  ``faces`` (F, 3) int64 or int32 is shared by every view.  Each face is
    subdivided at its edges' midpoints while its longest squared edge exceeds
    ``((resolution - 1) / resolution**2)**2``, with the reference's rounding; every vertex and every
    midpoint made sets voxel ``round(p * (resolution - 1))`` when it lies in the grid.  As in the
    reference, a face with a NaN coordinate is not split and a NaN point is dropped.

    Returns a (B, resolution, resolution, resolution) tensor of 0 and 1 in the normalised points'
    dtype, equal to the reference bit for bit; with ``return_sparse`` a ``sparse_coo`` tensor, its
    indices in sorted (view, x, y, z) order, values ones, not marked coalesced.  All views go
    through one launch per kernel and the call reads back one status (with the sparse size).

    Deliberate deviations from the reference:

    - a face or sub-triangle with an infinite coordinate is not split (its finite vertices still
      count); the reference does not return on such input;
    - a face index outside ``[0, V)`` raises IndexError (the reference asserts on the device);
    - a face that needs more than ``MAX_DEPTH`` (24) levels of subdivision (estimated from its longest edge, for
      faces that reach into the grid) raises ValueError;
    - ``resolution < 2`` raises ValueError where the reference asserts;
    - a batch of 0 views returns an empty grid (the reference raises in ``torch.cat``);
    - only float32 and float64 normalised points are accepted (TypeError otherwise), and there is no
      CPU path (a CPU tensor raises NotImplementedError).
    """
    func = "trianglemeshes_to_voxelgrids"
    _check_resolution(func, resolution, 2)
    _check_points(func, "vertices", vertices)
    if not isinstance(faces, torch.Tensor) or faces.dtype not in (torch.int64, torch.int32):
        raise TypeError(f"{func}: expected faces to be an int64 or int32 tensor")
    if faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f"{func}: expected faces of shape (num_faces, 3), got {list(faces.shape)}")
    if faces.device != vertices.device:
        raise ValueError(f"{func}: faces are on {faces.device}, vertices on {vertices.device}")
    points = _normalize(vertices, origin, scale)
    return _voxelize(func, points, faces.to(torch.int64).contiguous(), resolution, return_sparse)

