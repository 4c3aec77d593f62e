"""TEST ORACLE — ``voxelgrids_to_cubic_meshes`` restated in numpy from its contract (kaolin_b200/csrc/cubic_meshes.cu).

One view (X, Y, Z) is read as float32 and padded with zeros; its corner lattice is (X+1, Y+1, Z+1).
Face (a, p) lies between voxel p and voxel p - e_a and exists when p is inside the grid on the other
two axes and d = rint(v(p) - v(p - e_a)) != 0 (float32, half to even, NaN != 0).  Its quad is
[p, p + e_b, p + e_b + e_c, p + e_c], b = (a+1) mod 3, c = (a+2) mod 3, reversed when d < 0.  Faces
go axis by axis, each in lattice order; as triangles, every quad's [q0, q3, q1] and then every quad's
[q2, q1, q3].  The vertices are the used lattice points in lattice order.  Vectorised: a 128^3 view
takes about a second.
"""
import numpy as np


def extract(grid, is_trimesh=True):
    """grid (X, Y, Z) -> (vertices (nv, 3) float32, faces (nf, 3 or 4) int64)."""
    g = np.asarray(grid).astype(np.float32)
    X, Y, Z = g.shape
    dims = (X, Y, Z)
    pad = np.zeros((X + 2, Y + 2, Z + 2), np.float32)
    pad[1:-1, 1:-1, 1:-1] = g                       # voxel p at pad[p + 1]
    lat = (X + 1, Y + 1, Z + 1)
    here = pad[1:, 1:, 1:]                          # voxel p for every lattice point p
    quads, flips = [], []
    for a in range(3):
        lo = [slice(1, None)] * 3
        lo[a] = slice(0, X + 1 if a == 0 else Y + 1 if a == 1 else Z + 1)
        with np.errstate(invalid="ignore", over="ignore"):
            d = np.rint(here - pad[tuple(lo)])
            keep = ~(d == 0)
            rev = d < 0
        b, c = (a + 1) % 3, (a + 2) % 3
        inside = np.ones(lat, bool)
        for ax in (b, c):
            sl = [slice(None)] * 3
            sl[ax] = dims[ax]
            inside[tuple(sl)] = False
        keep &= inside
        p = np.stack(np.nonzero(keep), 1).astype(np.int64)
        eb, ec = np.eye(3, dtype=np.int64)[b], np.eye(3, dtype=np.int64)[c]
        quads.append(np.stack([p, p + eb, p + eb + ec, p + ec], 1))
        flips.append(rev[keep])
    q = np.concatenate(quads, 0)                    # (nq, 4, 3)
    flip = np.concatenate(flips, 0)
    q[flip] = q[flip][:, ::-1]
    flat = (q[..., 0] * lat[1] + q[..., 1]) * lat[2] + q[..., 2]
    used = np.zeros(lat[0] * lat[1] * lat[2], bool)
    used[flat.reshape(-1)] = True
    ids = np.cumsum(used) - 1
    verts = np.stack(np.unravel_index(np.nonzero(used)[0], lat), 1).astype(np.float32)
    faces = ids[flat].astype(np.int64)
    if is_trimesh:
        faces = np.concatenate([faces[:, [0, 3, 1]], faces[:, [2, 1, 3]]], 0)
    return verts.reshape(-1, 3), faces.reshape(-1, 3 if is_trimesh else 4)


def cubic_meshes(grids, is_trimesh=True):
    """grids (B, X, Y, Z) -> two lists of B arrays, as ``voxelgrids_to_cubic_meshes`` returns them."""
    out = [extract(g, is_trimesh) for g in grids]
    return [v for v, _ in out], [f for _, f in out]
