"""kaolin.ops.voxelgrid on sm_90a kernels (csrc/voxelgrid.cu): ``fill``, ``extract_surface``,
``extract_odms``, ``project_odms`` and ``downsample``.

The reference fills on the host, one ``scipy.ndimage.binary_fill_holes`` call per view, and raises for
a CUDA tensor; its other three operators are chains of torch passes with (B, 2, X, Y, Z) int64 or
broadcast uint8 temporaries.  Here every view goes through one launch of each kernel, no function
reads anything back to the host, and the output shapes follow from the input shapes.
"""
import torch
import torch.nn.functional as F

from .. import _lib
from .conversions.voxelgrid import _native

__all__ = ["downsample", "extract_surface", "fill", "extract_odms", "project_odms"]

_SURFACE_DTYPES = {torch.bool: _lib.DTYPE_U8, torch.float32: _lib.DTYPE_F32, torch.float64: _lib.DTYPE_F64}
_ODM_DTYPES = {torch.int64: _lib.DTYPE_I64, torch.int32: _lib.DTYPE_I32, torch.float32: _lib.DTYPE_F32,
               torch.float64: _lib.DTYPE_F64}
_PROJECT_GRID_DTYPES = {torch.bool: _lib.DTYPE_BOOL, torch.uint8: _lib.DTYPE_U8, torch.float32: _lib.DTYPE_F32,
                        torch.float64: _lib.DTYPE_F64}


def _check_grid(func, voxelgrids):
    if not voxelgrids.is_cuda:
        raise NotImplementedError(f"{func} does not support CPU.")
    if voxelgrids.ndim != 4:
        raise ValueError(f"Expected voxelgrids to have 4 dimensions but got {voxelgrids.ndim} dimensions.")


def _occupancy(voxelgrids):
    """(dtype flag, tensor the kernels read) for an occupancy test of any dtype: bool, uint8 and float32
    in place, anything else as ``voxelgrids != 0``."""
    if voxelgrids.dtype not in (torch.bool, torch.uint8, torch.float32):
        voxelgrids = voxelgrids != 0
    return _native(voxelgrids)


def _force_float(voxelgrids):
    """The reference's cast for pooling: bool to float16 on CUDA, anything else unchanged."""
    return voxelgrids.half() if voxelgrids.dtype == torch.bool else voxelgrids


def downsample(voxelgrids, scale):
    r"""kaolin.ops.voxelgrid.downsample: ``avg_pool3d`` of each view with kernel and stride ``scale`` (an
    int, or a list of three), not thresholded.  Plain torch, as in the reference, with its errors; there
    is no CPU path (a CPU tensor raises NotImplementedError)."""
    if not voxelgrids.is_cuda:
        raise NotImplementedError("downsample does not support CPU.")
    voxelgrids = _force_float(voxelgrids)
    try:
        output = F.avg_pool3d(voxelgrids.unsqueeze(1), kernel_size=scale, stride=scale, padding=0)
    except RuntimeError as err:
        if isinstance(scale, list) and len(scale) != 3:
            raise ValueError(f"Expected scale to have 3 dimensions but got {len(scale)} dimensions.")
        if voxelgrids.ndim != 4:
            raise ValueError(f"Expected voxelgrids to have 4 dimensions but got {voxelgrids.ndim} dimensions.")
        for i in range(3):
            if scale[i] < 1:
                raise ValueError(f"Downsample ratio must be at least 1 along every dimension but got {scale[i]} "
                                 f"at index {i}.")
            if scale[i] > voxelgrids.shape[i + 1]:
                raise ValueError(f"Downsample ratio must be less than voxelgrids shape of "
                                 f"{voxelgrids.shape[i + 1]} at index {i}, but got {scale[i]}.")
        raise err
    except TypeError as err:
        if not isinstance(scale, list) and not isinstance(scale, int):
            raise TypeError(f"Expected scale to be type list or int but got {type(scale)}.")
        raise err
    return output.squeeze(1)


def extract_surface(voxelgrids, mode="wide"):
    r"""kaolin.ops.voxelgrid.extract_surface: the occupied voxels of ``voxelgrids`` (B, X, Y, Z) with an
    empty or outside neighbour, as bool (B, X, Y, Z).

    ``"wide"`` keeps a voxel that is nonzero and whose mean over its zero-padded 3x3x3 window is below
    1; ``"thin"`` one whose mean over any of its three 3-voxel axis windows is.  For bool grids that is:
    occupied, with one of its 26 (thin: 6 face) neighbours empty or outside the grid.  float32 and
    float64 grids sum the window in their own dtype in the order of torch's CUDA ``avg_pool3d`` and
    divide with its rounding, so the result is bit-equal to the reference's on the GPU for any values.
    One launch for all views; strided grids are read in place.

    Deliberate deviations from the reference:

    - float16 and bfloat16 grids raise ``TypeError`` (the reference pools them in their own dtype);
      integer grids raise ``TypeError`` too, where the reference fails inside ``avg_pool3d``;
    - grids with a side below 3 are served, where ``avg_pool3d`` raises;
    - there is no CPU path (a CPU tensor raises NotImplementedError).
    """
    func = "extract_surface"
    _check_grid(func, voxelgrids)
    if mode not in ("wide", "thin"):
        raise ValueError(f'mode "{mode}" is not supported.')
    if voxelgrids.dtype not in _SURFACE_DTYPES:
        raise TypeError(f"{func}: expected a bool, float32 or float64 grid, got {voxelgrids.dtype}")
    B, X, Y, Z = voxelgrids.shape
    out = torch.empty((B, X, Y, Z), dtype=torch.bool, device=voxelgrids.device)
    if out.numel() == 0:
        return out
    g = voxelgrids.view(torch.uint8) if voxelgrids.dtype == torch.bool else voxelgrids
    _lib.call("dibr_b200_voxelgrid_extract_surface", g.device, B, X, Y, Z, _SURFACE_DTYPES[voxelgrids.dtype],
              int(mode == "thin"), g, *g.stride(), out, what=func)
    return out


def fill(voxelgrids):
    r"""kaolin.ops.voxelgrid.fill: ``voxelgrids`` (B, X, Y, Z) with its holes filled, as bool (B, X, Y, Z).

    A voxel is occupied when its value is nonzero (NaN is, -0.0 is not).  The output is true where the
    voxel is occupied, or where it is empty and its 6-connected component of empty voxels touches none
    of the six border faces: ``scipy.ndimage.binary_fill_holes`` with its default structure.  A cavity
    reached from the border only through edge- or corner-diagonal steps is filled.  Bool, uint8 and
    float32 grids are read in place, strided or not; other dtypes go through ``voxelgrids != 0``.

    The kernels label each view's empty voxels with a union-find (csrc/voxelgrid.cu): three launches for
    all views whatever the content, no host read, and 4 bytes of workspace per voxel.  The result does
    not depend on the order the atomics run in, so reruns are byte-identical.  Each view must hold fewer
    than 2^31 - 1 voxels (else RuntimeError); the batch may be of any size.  Not differentiable.

    Deliberate deviations from the reference:

    - CUDA input is served, where the reference raises NotImplementedError;
    - CPU input raises NotImplementedError, where the reference runs scipy;
    - B = 0 returns an empty bool tensor, where the reference raises in ``torch.stack``;
    - a side of 0 returns an empty tensor.
    """
    func = "fill"
    _check_grid(func, voxelgrids)
    B, X, Y, Z = voxelgrids.shape
    dev = voxelgrids.device
    nbytes = _lib.voxelgrid_fill_workspace_bytes(B, X, Y, Z, func)
    out = torch.empty((B, X, Y, Z), dtype=torch.bool, device=dev)
    if out.numel() == 0:
        return out
    flag, g = _occupancy(voxelgrids)
    _lib.call("dibr_b200_voxelgrid_fill", dev, B, X, Y, Z, flag, g, *g.stride(), out, _lib.scratch(nbytes, dev),
              nbytes, what=func)
    return out


def extract_odms(voxelgrids):
    r"""kaolin.ops.voxelgrid.extract_odms: the six orthographic depth maps of ``voxelgrids`` (B, dim, dim,
    dim), as int64 (B, 6, dim, dim), in the face order z_neg, z_pos, y_neg, y_pos, x_neg, x_pos.

    Each entry counts the empty voxels on its ray before the first occupied one from that side, or is
    ``dim`` when there is none.  Maps 0 and 1 are indexed [x, y], maps 2 and 3 [x, z], maps 4 and 5
    [y, z].  Occupancy is ``.bool()`` (NaN is occupied).  Bool, uint8 and float32 grids are read in place;
    other dtypes go through ``voxelgrids != 0``.  The grid is read once for all six maps, with integer
    atomics whose order does not change the result; no host read.

    Deliberate deviations from the reference:

    - a non-cubic grid raises ``ValueError`` (the reference fails inside a broadcast);
    - there is no CPU path (a CPU tensor raises NotImplementedError).
    """
    func = "extract_odms"
    _check_grid(func, voxelgrids)
    B, X, Y, Z = voxelgrids.shape
    if not X == Y == Z:
        raise ValueError(f"{func}: expected a cubic grid (batch_size, dim, dim, dim), got {list(voxelgrids.shape)}")
    out = torch.empty((B, 6, Z, Z), dtype=torch.int64, device=voxelgrids.device)
    if B * Z == 0:
        return out
    flag, g = _occupancy(voxelgrids)
    _lib.call("dibr_b200_voxelgrid_extract_odms", g.device, B, Z, flag, g, *g.stride(), out, what=func)
    return out


def project_odms(odms, voxelgrids=None, votes=1):
    r"""kaolin.ops.voxelgrid.project_odms: carve ``voxelgrids`` (B, dim, dim, dim) with the orthographic
    depth maps ``odms`` (B, 6, dim, dim); without a grid, a full one.  Returns bool (B, dim, dim, dim).

    Per voxel (x, y, z) the six masks ``z >= dim - odms[0][x, y]``, ``z < odms[1][x, y]`` and the same
    over y (maps 2, 3 at [x, z]) and x (maps 4, 5 at [y, z]) are counted, and the output is
    ``voxel * votes - count > 0``.  ``dim - odm`` is computed in the dtype of ``odms`` (int64, int32,
    float32 or float64; fractional float maps are accepted) and compared with the index as torch's
    type promotion does.  The arithmetic is the reference's: int64 for bool grids and the default full
    grid, float32 or float64 for float grids and **uint8, wrapping, for uint8 grids**, so there a voxel
    of 1 with ``votes = 1`` and two masks gives 255 and stays true.  One launch; no host read.

    Deliberate deviations from the reference:

    - odms and grids of other dtypes raise ``TypeError``; ``votes`` must be an int;
    - there is no CPU path (a CPU tensor raises NotImplementedError).
    """
    func = "project_odms"
    if not odms.is_cuda:
        raise NotImplementedError(f"{func} does not support CPU.")
    if odms.ndim != 4 or odms.shape[1] != 6:
        shape1 = odms.shape[1] if odms.ndim > 1 else None
        raise ValueError(f"Expected odms' second dimension to be 6, but got {shape1} instead.")
    B, _, D0, D = odms.shape
    if D0 != D:
        raise ValueError(f"{func}: expected odms of shape (batch_size, 6, dim, dim), got {list(odms.shape)}")
    if odms.dtype not in _ODM_DTYPES:
        raise TypeError(f"{func}: expected int64, int32, float32 or float64 odms, got {odms.dtype}")
    if isinstance(votes, bool) or not isinstance(votes, int):
        raise TypeError(f"{func}: expected votes to be an int, got {type(votes)}")
    dev = odms.device
    if voxelgrids is None:
        gflag, g, strides = _lib.VOXELGRID_ALL_ONES, None, (0, 0, 0, 0)
    else:
        if voxelgrids.ndim != 4:
            raise ValueError(f"Expected voxelgrids to have 4 dimensions but got {voxelgrids.ndim} dimensions.")
        if voxelgrids.shape[0] != B:
            raise ValueError(f"Expected voxelgrids and odms' batch size to be the same, but got {B} for odms and "
                             f"{voxelgrids.shape[0]} for voxelgrid.")
        for i in voxelgrids.shape[1:]:
            if i != D:
                raise ValueError(f"Expected voxelgrids and odms' dimension size to be the same, but got {D} for "
                                 f"odms and {i} for voxelgrid.")
        if voxelgrids.device != dev:
            raise ValueError(f"{func}: odms are on {dev} and voxelgrids on {voxelgrids.device}")
        if voxelgrids.dtype not in _PROJECT_GRID_DTYPES:
            raise TypeError(f"{func}: expected a bool, uint8, float32 or float64 grid, got {voxelgrids.dtype}")
        gflag = _PROJECT_GRID_DTYPES[voxelgrids.dtype]
        g = voxelgrids.view(torch.uint8) if voxelgrids.dtype == torch.bool else voxelgrids
        strides = g.stride()
    out = torch.empty((B, D, D, D), dtype=torch.bool, device=dev)
    if out.numel() == 0:
        return out
    o = odms.contiguous()
    _lib.call("dibr_b200_voxelgrid_project_odms", dev, B, D, _ODM_DTYPES[odms.dtype], o, gflag, g, *strides, votes,
              out, what=func)
    return out
