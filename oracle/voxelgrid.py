"""TEST INFRASTRUCTURE — a numpy restatement of kaolin.ops.voxelgrid's fill, extract_surface,
extract_odms and project_odms (kaolin_b200/ops/voxelgrid.py), written from their definitions:

- fill: a breadth-first flood of the empty voxels from the six border faces under 6-connectivity;
  everything the flood does not reach is filled;
- extract_surface: the zero-padded window sums in the grid's float dtype (x outer, z inner), divided
  in that dtype and compared with 1; bool grids count occupied neighbours;
- extract_odms: the first and last occupied voxel of every axis ray;
- project_odms: the six masks and ``voxel * votes - count > 0`` in the reference's result dtype.
"""
import numpy as np


def occupied(grid):
    """Nonzero, as numpy's truthiness: NaN is occupied, -0.0 is not."""
    return np.asarray(grid) != 0


def fill(grid):
    """(B, X, Y, Z) of any dtype -> bool (B, X, Y, Z)."""
    occ = occupied(grid)
    out = np.empty(occ.shape, bool)
    for b in range(occ.shape[0]):
        empty = ~occ[b]
        reached = np.zeros_like(empty)
        front = np.zeros_like(empty)
        for ax in range(3):
            for end in (0, -1):
                idx = [slice(None)] * 3
                idx[ax] = end
                front[tuple(idx)] |= empty[tuple(idx)]
        while front.any():
            reached |= front
            nxt = np.zeros_like(front)
            nxt[1:] |= front[:-1]
            nxt[:-1] |= front[1:]
            nxt[:, 1:] |= front[:, :-1]
            nxt[:, :-1] |= front[:, 1:]
            nxt[:, :, 1:] |= front[:, :, :-1]
            nxt[:, :, :-1] |= front[:, :, 1:]
            front = nxt & empty & ~reached
        out[b] = ~reached
    return out


def extract_surface(grid, mode="wide"):
    """(B, X, Y, Z) bool, float32 or float64 -> bool (B, X, Y, Z)."""
    g = np.asarray(grid)
    occ = occupied(g)
    if g.dtype == bool:
        v, n_wide, n_thin = g.astype(np.int64), 27, 3
        below = lambda s, n: s < n
    else:
        v = g
        below = lambda s, n: (s / g.dtype.type(n)) < 1
    p = np.pad(v, ((0, 0), (1, 1), (1, 1), (1, 1)))
    X, Y, Z = g.shape[1:]
    win = lambda dx, dy, dz: p[:, 1 + dx:1 + dx + X, 1 + dy:1 + dy + Y, 1 + dz:1 + dz + Z]
    zero = np.zeros(g.shape, v.dtype)
    if mode == "wide":
        s = zero.copy()
        for dx in (-1, 0, 1):
            for dy in (-1, 0, 1):
                for dz in (-1, 0, 1):
                    s = s + win(dx, dy, dz)
        return below(s, 27) & occ
    sx, sy, sz = zero.copy(), zero.copy(), zero.copy()
    for d in (-1, 0, 1):
        sx = sx + win(d, 0, 0)
        sy = sy + win(0, d, 0)
        sz = sz + win(0, 0, d)
    return (below(sx, 3) | below(sy, 3) | below(sz, 3)) & occ


def extract_odms(grid):
    """(B, D, D, D) of any dtype -> int64 (B, 6, D, D)."""
    occ = occupied(grid)
    D = occ.shape[-1]
    out = []
    for ax in (3, 2, 1):
        any_ = occ.any(axis=ax)
        first = np.where(any_, occ.argmax(axis=ax), D)
        last = np.where(any_, D - 1 - np.flip(occ, axis=ax).argmax(axis=ax), -1)
        out += [D - 1 - last, first]
    return np.stack(out, 1).astype(np.int64)


def project_odms(odms, grid=None, votes=1):
    """odms (B, 6, D, D) int64, int32, float32 or float64; grid (B, D, D, D) bool, uint8, float32,
    float64 or None -> bool (B, D, D, D)."""
    odms = np.asarray(odms)
    B, _, _, D = odms.shape
    with np.errstate(over="ignore"):
        pos = odms.copy()
        pos[:, 0::2] = (odms.dtype.type(D) - odms[:, 0::2]).astype(odms.dtype)
    idx = np.arange(D)
    if odms.dtype.kind == "f":
        idx = idx.astype(odms.dtype)
        cmp = pos
    else:
        cmp = pos.astype(np.int64)
    i_x = idx[None, :, None, None]
    i_y = idx[None, None, :, None]
    i_z = idx[None, None, None, :]
    count = ((i_z >= cmp[:, 0, :, :, None]).astype(np.int64) + (i_z < cmp[:, 1, :, :, None])
             + (i_y >= cmp[:, 2, :, None, :]) + (i_y < cmp[:, 3, :, None, :])
             + (i_x >= cmp[:, 4, None, :, :]) + (i_x < cmp[:, 5, None, :, :]))
    if grid is None:
        return (votes - count) > 0
    g = np.asarray(grid)
    if g.dtype == bool:
        return (g.astype(np.int64) * votes - count) > 0
    if g.dtype == np.uint8:
        return ((g.astype(np.int64) * votes - count) % 256) != 0
    t = g.dtype.type
    with np.errstate(invalid="ignore"):
        return (g * t(votes) - count.astype(g.dtype)) > 0
