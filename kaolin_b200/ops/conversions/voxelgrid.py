"""kaolin.ops.conversions.voxelgrids_to_trianglemeshes and voxelgrids_to_cubic_meshes on sm_90a kernels
(csrc/marching_cubes.cu, csrc/cubic_meshes.cu).

The reference (voxelgrid.py:158-246) loops over the views in Python: each costs a ``torch.all``
sync, a padded float copy, six device-to-host copies, a device synchronise and about 112 bytes of
zero-filled scratch per padded voxel.  Here every view goes through one launch per kernel: classify
and count every (view, cube), scan the counts once for all views, read back the per-view totals (the
call's one device-to-host read) and write every view's vertices and faces in one kernel.  The zero
border the reference pads with is virtual: the kernels sample around the grid, nothing is copied.
"""
import torch

from ... import _lib
from ...render.mesh import _host

__all__ = ["voxelgrids_to_trianglemeshes", "voxelgrids_to_cubic_meshes", "unbatched_mcube_forward"]


def case_table():
    """(256, 5, 3, 2) int32: for each case sum_k (field(corner k) < iso) 2^k, the corner pairs (i, j)
    whose edges hold the vertices of each triangle, in the published table's order; -1 past the
    case's triangles.  Corners use the reference's numbering (csrc/marching_cubes.cu)."""
    return torch.tensor(_lib.marching_cubes_case_table(), dtype=torch.int32).view(256, 5, 3, 2)


def _native(grid):
    """(dtype flag, tensor the kernels read): float32 and uint8 as they are, bool as its bytes."""
    if grid.dtype == torch.float32:
        return _lib.DTYPE_F32, grid
    if grid.dtype == torch.uint8:
        return _lib.DTYPE_U8, grid
    if grid.dtype == torch.bool:
        return _lib.DTYPE_U8, grid.view(torch.uint8)
    raise AssertionError(grid.dtype)


class _Emit(torch.autograd.Function):
    """grid (B, X, Y, Z) -> the vertices of every view in one (sum nv, 3) tensor; fills ``faces``."""

    @staticmethod
    def forward(ctx, grid, lattice, iso, cases, scan, num_vertices, faces):
        ctx.set_materialize_grads(False)
        B, X, Y, Z, pad = lattice
        dev = grid.device
        flag, g = _native(grid)
        verts = torch.empty((num_vertices, 3), dtype=torch.float32, device=dev)
        if faces.numel():
            _lib.call("dibr_b200_marching_cubes_emit", dev, B, X, Y, Z, pad, flag, g, *g.stride(), iso, cases, scan,
                      verts if num_vertices else _lib.scratch(16, dev), faces, what="voxelgrids_to_trianglemeshes")
        ctx.lattice, ctx.iso, ctx.num_vertices = lattice, iso, num_vertices
        ctx.save_for_backward(grid, cases, scan)
        return verts

    @staticmethod
    def backward(ctx, grad):
        grid, cases, scan = ctx.saved_tensors
        if grad is None or not ctx.needs_input_grad[0]:
            return None, None, None, None, None, None, None
        if ctx.num_vertices == 0:
            return torch.zeros_like(grid), None, None, None, None, None, None
        B, X, Y, Z, pad = ctx.lattice
        out = torch.empty((B, X, Y, Z), dtype=torch.float32, device=grid.device)
        _lib.call("dibr_b200_marching_cubes_backward", grid.device, B, X, Y, Z, pad, grid, *grid.stride(), ctx.iso,
                  cases, scan, grad.contiguous(), out, what="voxelgrids_to_trianglemeshes")
        return out, None, None, None, None, None, None


def _march(func, grid, iso_value, pad):
    """grid (B, X, Y, Z) of a dtype the kernels read -> (flat vertices, flat faces, per-view vertex and
    face counts)."""
    B, X, Y, Z = grid.shape
    dev = grid.device
    iso = float(iso_value)
    nbytes = _lib.marching_cubes_workspace_bytes(B, X, Y, Z, pad, func)
    N = (X + 2 * pad) * (Y + 2 * pad) * (Z + 2 * pad)
    flag, g = _native(grid)
    cases = torch.empty(max(B * N, 1), dtype=torch.uint8, device=dev)
    scan = torch.empty(2 * (B * N + 1), dtype=torch.int32, device=dev)
    totals = torch.empty((B, 2), dtype=torch.int32, device=dev)
    _lib.call("dibr_b200_marching_cubes_count", dev, B, X, Y, Z, pad, flag, g, *g.stride(), iso, cases, scan, totals,
              _lib.scratch(nbytes, dev), nbytes, what=func)
    totals = totals.tolist()                          # the call's one device-to-host read
    nf = [t[0] for t in totals]
    nv = [t[1] for t in totals]
    faces = torch.empty((sum(nf), 3), dtype=torch.int64, device=dev)
    verts = _Emit.apply(grid, (B, X, Y, Z, pad), iso, cases, scan, sum(nv), faces)
    return verts, faces, nv, nf


def voxelgrids_to_trianglemeshes(voxelgrids, iso_value=0.5):
    r"""kaolin.ops.conversions.voxelgrids_to_trianglemeshes: marching cubes (Lorensen and Cline) on each
    view of ``voxelgrids`` (B, X, Y, Z), padded with a border of zeros.

    Returns ``(vertices, faces)``, two lists of B tensors: vertices (nv, 3) float32 in padded-grid
    units and in dim order, faces (nf, 3) int64, bit-equal to the reference wherever it is correct.
    A corner is inside when its value is below ``iso_value`` (NaN and values equal to it are outside).
    uint8, bool and float32 grids are read as they are, contiguous or not; other dtypes go through
    ``.float()``, as in the reference.  All views go through one launch per kernel, and the call makes
    one device-to-host read (the per-view counts).  If ``voxelgrids`` requires grad, the vertices carry
    autograd to it through t = (iso - f0) / (f1 - f0) on each vertex's edge; the backward makes no host
    read and uses no atomics, so its results are bit-reproducible.

    Deliberate deviations from the reference:

    - every voxel is processed: the reference's launch rounds its grid down and skips the last
      voxels (inputs of side 4 and 5, and of side 202 and more, lose part of their surface there);
    - non-cubic grids are extracted on their true axes (the reference strides them as if cubic);
    - there is no vertex cap (the reference drops vertices past X*Y*100 - 3 of the padded grid and
      leaves faces pointing at them);
    - a grid with no surface returns empty tensors and prints nothing;
    - the vertices have gradients, where the reference's backward returns None;
    - there is no CPU path, as in the reference (a CPU tensor raises NotImplementedError).
    """
    func = "voxelgrids_to_trianglemeshes"
    if not voxelgrids.is_cuda:
        raise NotImplementedError("voxelgrids_to_trianglemeshes does not support CPU.")
    if voxelgrids.dim() != 4:
        raise ValueError(f"{func}: expected voxelgrids of shape (batch_size, X, Y, Z), got {list(voxelgrids.shape)}")
    B = voxelgrids.shape[0]
    if B == 0:
        return [], []
    dev = voxelgrids.device
    if 0 in voxelgrids.shape[1:]:
        empty_v = [torch.zeros((0, 3), dtype=torch.float32, device=dev) for _ in range(B)]
        return empty_v, [torch.zeros((0, 3), dtype=torch.int64, device=dev) for _ in range(B)]
    grid = voxelgrids if voxelgrids.dtype in (torch.float32, torch.uint8, torch.bool) else voxelgrids.float()
    verts, faces, nv, nf = _march(func, grid, iso_value, 1)
    return list(torch.split(verts, nv)), list(torch.split(faces, nf))


def voxelgrids_to_cubic_meshes(voxelgrids, is_trimesh=True):
    r"""kaolin.ops.conversions.voxelgrids_to_cubic_meshes: "Cubify" (Mesh R-CNN, ICCV 2019) on each view
    of ``voxelgrids`` (B, X, Y, Z): every occupied voxel becomes a unit cube, and only the faces between
    occupied and empty space are kept.

    Returns ``(vertices, faces)``, two lists of B tensors: vertices (nv, 3) float32, the cube corners
    the faces use in lattice order, and faces int64 indices into them, (nf, 3) triangles when
    ``is_trimesh`` else (nq, 4) quads.  Wherever every voxel difference rounds to -1, 0 or 1 (every
    binary grid of any dtype and every float grid with values in [0, 1]) the output equals the
    reference's bit for bit.  Values are read as float32 and padded with zeros; a face lies between
    two voxels whose difference rounds (half to even) to nonzero, NaN included, and its winding
    follows the difference's sign (csrc/cubic_meshes.cu states the order).  uint8, bool and float32
    grids are read as they are, contiguous or not; other dtypes go through ``.float()``.  All views
    go through one launch per kernel, and the call makes one device-to-host read (the per-view
    counts).  The output is not differentiable, as in the reference: its vertices are lattice points.

    Deliberate deviations from the reference:

    - a face whose difference rounds to 2 or more in magnitude (a uint8 grid of 0 and 255, values
      above 1.5, infinities) is wound by the sign of the difference; the reference reverses only a
      difference of exactly -1, so it winds the far side of such a solid inward;
    - a batch whose every view is empty returns B pairs of empty tensors, vertices (0, 3) float32 and
      faces (0, 3) or (0, 4) int64, where the reference raises;
    - B = 0 returns ``([], [])``, and a grid with a zero-size axis returns B pairs of empty tensors;
    - there is no CPU path (a CPU tensor raises NotImplementedError, as in the other voxel operators),
      where the reference runs on the CPU;
    - an input that is not 4-D raises ValueError.
    """
    func = "voxelgrids_to_cubic_meshes"
    if not voxelgrids.is_cuda:
        raise NotImplementedError(f"{func} does not support CPU.")
    if voxelgrids.dim() != 4:
        raise ValueError(f"{func}: expected voxelgrids of shape (batch_size, X, Y, Z), got {list(voxelgrids.shape)}")
    B, X, Y, Z = voxelgrids.shape
    if B == 0:
        return [], []
    dev = voxelgrids.device
    corners = 3 if is_trimesh else 4
    if 0 in (X, Y, Z):
        empty_v = [torch.zeros((0, 3), dtype=torch.float32, device=dev) for _ in range(B)]
        return empty_v, [torch.zeros((0, corners), dtype=torch.int64, device=dev) for _ in range(B)]
    nbytes = _lib.cubic_meshes_workspace_bytes(B, X, Y, Z, func)
    native = voxelgrids.dtype in (torch.float32, torch.uint8, torch.bool)
    flag, g = _native(voxelgrids if native else voxelgrids.float())
    ws = _lib.scratch(nbytes, dev)
    totals = torch.empty((B, 2), dtype=torch.int32, device=dev)
    _lib.call("dibr_b200_cubic_meshes_count", dev, B, X, Y, Z, flag, g, *g.stride(), totals, ws, nbytes, what=func)
    totals = totals.tolist()                          # the call's one device-to-host read
    per_quad = 2 if is_trimesh else 1
    nf = [per_quad * t[0] for t in totals]
    nv = [t[1] for t in totals]
    verts = torch.empty((sum(nv), 3), dtype=torch.float32, device=dev)
    faces = torch.empty((sum(nf), corners), dtype=torch.int64, device=dev)
    if faces.numel():
        _lib.call("dibr_b200_cubic_meshes_emit", dev, B, X, Y, Z, int(bool(is_trimesh)), verts, faces, ws, nbytes,
                  what=func)
    return list(torch.split(verts, nv)), list(torch.split(faces, nf))


def unbatched_mcube_forward(voxelgrid, iso_value):
    """``_C.ops.conversions.unbatched_mcube_forward_cuda``: marching cubes on one already-padded grid
    (X, Y, Z) float32, sampled with the reference's clamp at the far border and no further padding.
    Returns ``[vertices (nv, 3) float32, faces (nf, 3) int32]``, without autograd.  A face corner on an
    edge of the grid's border that no cube owns (where the reference reads outside its buffers) is -1;
    grids padded as the reference's wrapper pads them have none."""
    func = "unbatched_mcube_forward_cuda"
    _host.check_tensors(func, [("voxelgrid", voxelgrid)], dtype=None)
    if voxelgrid.dtype != torch.float32:
        raise RuntimeError(f"{func}: expected scalar type Float but found "
                           f"{str(voxelgrid.dtype).replace('torch.', '').capitalize()}")
    if voxelgrid.dim() != 3:
        raise RuntimeError(f"{func}: expected voxelgrid of shape (X, Y, Z), got {list(voxelgrid.shape)}")
    dev = voxelgrid.device
    if voxelgrid.numel() == 0:
        return [torch.zeros((0, 3), dtype=torch.float32, device=dev), torch.zeros((0, 3), dtype=torch.int32, device=dev)]
    with torch.no_grad():
        verts, faces, _, _ = _march(func, voxelgrid.unsqueeze(0), iso_value, 0)
    return [verts, faces.int()]
