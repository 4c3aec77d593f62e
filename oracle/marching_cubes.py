"""TEST INFRASTRUCTURE — a numpy / torch restatement of the reference's marching cubes
(kaolin/ops/conversions/voxelgrid.py:158-246 and csrc/ops/conversions/unbatched_mcube), in two modes:
corrected (true axes, every voxel, no vertex cap: the behaviour
kaolin_b200.ops.conversions.voxelgrids_to_trianglemeshes promises) and faithful (the reference
operator's dropped voxels, scrambled strides and vertex cap).

``extract`` runs one view in float32 with the reference's rounding (an IEEE division for
t = (iso - f0) / (f1 - f0), then p0 + (p1 - p0) t with one rounding: p1 - p0 is 0 or +-1, so numpy's
float32 product is exact and the sum rounds once, as the fma does).  ``vertices_f64`` recomputes the
same vertices in float64 torch with autograd to the grid.

The case table is not this repository's: ``case_table_from_golden`` reads it off the reference's own
outputs for the 256 corner configurations of a 2 x 2 x 2 grid (tests/golden/ref_cuda_mcube.npz),
where every vertex is an edge midpoint and each triangle's three edges lie on exactly one cube.
"""
import numpy as np
import torch

# The reference's corner and edge numbering (helper geometry, not its table): corner k at
# (x, y, z) = ((k ^ k >> 1) & 1, k >> 1 & 1, k >> 2 & 1), x the fastest (last) axis; edge e runs
# from EDGES[e][0] to EDGES[e][1].
EDGES = [(0, 1), (1, 2), (2, 3), (3, 0), (4, 5), (5, 6), (6, 7), (7, 4), (0, 4), (1, 5), (2, 6), (3, 7)]
OWNED = (6, 7, 11)      # the edges a cube writes vertices for: along x, y and z through corner 7


def corner_abc(k):
    """Corner k as an offset along the array's dims (a, b, c) = (z, y, x)."""
    return (k >> 2) & 1, (k >> 1) & 1, (k ^ (k >> 1)) & 1


def edge_owner(e):
    """(offset (da, db, dc) from a cube to the owner of its edge e, slot of e in the owner)."""
    i, j = EDGES[e]
    ci, cj = corner_abc(i), corner_abc(j)
    lo = [min(u, v) for u, v in zip(ci, cj)]
    if ci[2] != cj[2]:
        return (lo[0] - 1, lo[1] - 1, lo[2]), 0
    if ci[1] != cj[1]:
        return (lo[0] - 1, lo[1], lo[2]), 1
    return (lo[0], lo[1] - 1, lo[2]), 2


def _edge_of_midpoint(cube, mid):
    """The reference edge number of cube (a, b, c) whose midpoint is ``mid`` (in dim order)."""
    for e, (i, j) in enumerate(EDGES):
        m = [cube[d] + (corner_abc(i)[d] + corner_abc(j)[d]) / 2 for d in range(3)]
        if np.allclose(m, mid):
            return e
    return None


def case_table_from_golden(golden):
    """list of 256 edge lists (3 per triangle, in the table's order) from the reference's outputs
    ``golden[k] = (vertices, faces)`` on the 2 x 2 x 2 grid whose corner i (flat index a*4 + b*2 + c)
    holds bit i of k, padded by the wrapper: corner k of the middle cube (1, 1, 1) is that grid's
    point at corner_abc(k), so the middle cube's case is k with in = (value < 0.5) flipped."""
    table = []
    for k in range(256):
        verts, faces = golden[k]
        cs = 0
        for c in range(8):
            a, b, cc = corner_abc(c)
            cs |= (((k >> (a * 4 + b * 2 + cc)) & 1) == 0) << c
        table.append(None)
        tris = []
        for f in faces:
            edges = [_edge_of_midpoint((1, 1, 1), verts[v]) for v in f[::-1]]
            if None not in edges:
                tris += edges
        table[-1] = (cs, tris)
    out = [None] * 256
    for cs, tris in table:
        out[cs] = tris
    assert all(t is not None for t in out)
    return out


class Tables:
    """Per-case arrays derived from an edge table: triangle count, owned-vertex count and rank of
    each owned edge (first occurrence in the triangle list; -1 when absent)."""

    def __init__(self, table):
        self.table = table
        self.ntri = np.array([len(t) // 3 for t in table], np.int64)
        self.rank = np.full((256, 3), -1, np.int64)
        for cs, t in enumerate(table):
            n = 0
            for e in t:
                if e in OWNED and self.rank[cs, OWNED.index(e)] < 0:
                    self.rank[cs, OWNED.index(e)] = n
                    n += 1
        self.nown = (self.rank >= 0).sum(1)
        self.edges = np.full((256, 15), -1, np.int64)
        for cs, t in enumerate(table):
            self.edges[cs, :len(t)] = t


def launched_voxels(num_voxels):
    """The voxels the reference's classify and compact launches cover (unbatched_mcube_cuda.cu:157-173):
    ``grid.x = num_voxels / 128`` rounds down, and above 65535 CTAs the grid is re-cut as
    ``(32768, grid.x / 32768)``, rounding down again."""
    if num_voxels < 128:
        return num_voxels
    gx, gy = num_voxels // 128, 1
    if gx > 65535:
        gx, gy = 32768, gx // 32768
    return gx * gy * 128


def extract(grid, iso, tables, pad=1, faithful=False):
    """One view (X, Y, Z) -> (vertices (nv, 3) float32, faces (nf, 3) int64, topology).

    ``faithful=False`` is the corrected reference: every voxel, the grid's true axes, no cap.
    ``faithful=True`` reproduces the reference operator's quirks: the padded grid's memory read as if
    its last axis had the length of its first (a C array of shape (Z, Y, X)), neighbour cubes found by
    linear index arithmetic, the voxels past ``launched_voxels`` never classified (no triangles, and
    a vertex order of zeros), and the vertices cut to X*Y*100 rows, those from row X*Y*100 - 3 on
    never written (zeros).  Face
    corners the reference leaves undefined are -2 where the owner's vertex order lacks the edge (it
    reads an uninitialised offset) and -3 where the owner lies outside the grid (it reads outside
    its buffers).
    ``topology`` = (owner cube of each vertex, its slot, lattice shape), for vertices_f64."""
    grid = np.asarray(grid, np.float32)
    iso = np.float32(iso)
    g = np.pad(grid, pad) if pad else grid
    if faithful:
        g = np.ascontiguousarray(g).reshape(g.shape[::-1])
    E = np.pad(g, ((0, 1), (0, 1), (0, 1)), mode="edge")     # the far border, clamped
    NA, NB, NC = g.shape
    f = np.stack([E[da:da + NA, db:db + NB, dc:dc + NC] for da, db, dc in map(corner_abc, range(8))])
    case = np.zeros((NA, NB, NC), np.int64)
    for k in range(8):
        case |= (f[k] < iso).astype(np.int64) << k
    case = case.ravel()
    f = f.reshape(8, -1)
    N = case.size
    q = np.arange(N)
    live = q < (launched_voxels(N) if faithful else N)
    counted = np.where(live, case, 0)
    vscan = np.concatenate([[0], np.cumsum(tables.nown[counted])])
    tscan = np.concatenate([[0], np.cumsum(tables.ntri[counted])])
    nv, nf = int(vscan[-1]), int(tscan[-1])
    a, b, c = q // (NB * NC), (q // NC) % NB, q % NC
    verts = np.zeros((nv, 3), np.float32)
    own_q, own_s = np.zeros(nv, np.int64), np.zeros(nv, np.int64)
    p = np.stack([a, b, c], 1).astype(np.float32)
    with np.errstate(all="ignore"):
        for s, e in enumerate(OWNED):
            r = tables.rank[counted, s]
            sel = r >= 0
            k0, k1 = EDGES[e]
            f0, f1 = f[k0, sel], f[k1, sel]
            t = (iso - f0) / (f1 - f0)
            p0 = p[sel] + np.array(corner_abc(k0), np.float32)
            p1 = p[sel] + np.array(corner_abc(k1), np.float32)
            rows = vscan[q[sel]] + r[sel]
            verts[rows] = p0 + (p1 - p0) * t[:, None]
            own_q[rows], own_s[rows] = q[sel], s
    if faithful:       # the reference's vertex buffer has X*Y*100 rows, written below row X*Y*100 - 3
        verts = verts[:NC * NB * 100]
        verts[max(NC * NB * 100 - 3, 0):] = 0
    faces = np.zeros((nf, 3), np.int64)
    for t in range(5):
        sel = tables.ntri[counted] > t
        qs, cs = q[sel], counted[sel]
        for k in range(3):
            e = tables.edges[cs, 3 * t + k]
            ids = np.full(qs.size, -1, np.int64)
            for ed in range(12):
                m = e == ed
                (da, db, dc), s = edge_owner(ed)
                if faithful:
                    o = qs[m] + (da * NB + db) * NC + dc
                    inside = (o >= 0) & (o < N)
                    o = np.where(inside, o, 0)
                    rank = tables.rank[counted[o], s]
                    rank = np.where(tables.nown[counted[o]] == 0, 0, rank)
                    val = np.where(live[o] & (rank >= 0), vscan[o] + rank, -2)
                    val = np.where(inside, val, -3)
                else:
                    oa, ob, oc = a[qs[m]] + da, b[qs[m]] + db, c[qs[m]] + dc
                    ok = (oa >= 0) & (oa < NA) & (ob >= 0) & (ob < NB) & (oc >= 0) & (oc < NC)
                    o = (oa * NB + ob) * NC + oc
                    val = np.full(m.sum(), -1, np.int64)
                    val[ok] = vscan[o[ok]] + tables.rank[case[o[ok]], s]
                ids[m] = val
            faces[tscan[qs] + t, 2 - k] = ids
    return verts, faces, (own_q, own_s, (NA, NB, NC))


def vertices_f64(grid, iso, topology, pad=1):
    """The vertices of ``extract``'s topology in float64 torch, differentiable with respect to
    ``grid`` (a float64 tensor (X, Y, Z))."""
    own_q, own_s, (NA, NB, NC) = topology
    g = torch.nn.functional.pad(grid, (pad,) * 6) if pad else grid
    g = torch.nn.functional.pad(g[None, None], (0, 1, 0, 1, 0, 1), mode="replicate")[0, 0]
    q = torch.from_numpy(own_q).to(grid.device)
    s = torch.from_numpy(own_s).to(grid.device)
    a, b, c = q // (NB * NC), (q // NC) % NB, q % NC
    out = torch.zeros((len(q), 3), dtype=torch.float64, device=grid.device)
    for slot, e in enumerate(OWNED):
        m = s == slot
        k0, k1 = EDGES[e]
        d0, d1 = corner_abc(k0), corner_abc(k1)
        f0 = g[a[m] + d0[0], b[m] + d0[1], c[m] + d0[2]]
        f1 = g[a[m] + d1[0], b[m] + d1[1], c[m] + d1[2]]
        t = (iso - f0) / (f1 - f0)
        base = torch.stack([a[m], b[m], c[m]], 1).double()
        p0 = base + torch.tensor(d0, dtype=torch.float64, device=grid.device)
        p1 = base + torch.tensor(d1, dtype=torch.float64, device=grid.device)
        out = out.index_put((m.nonzero()[:, 0],), p0 + (p1 - p0) * t[:, None])
    return out


# Scenes of tests/golden/ref_cuda_mcube.npz: name -> (grid (B, X, Y, Z), iso value).  All cubic, of
# sides whose voxels the reference's launch covers, and below its vertex cap, where its output is
# correct.
def case_grids():
    """(256, 2, 2, 2) uint8: view k holds bit i of k at flat index i."""
    k = np.arange(256)[:, None]
    return ((k >> np.arange(8)[None, :]) & 1).astype(np.uint8).reshape(256, 2, 2, 2)


def sphere(n, center=(0.05, -0.1, 0.0)):
    """The distance of each grid point from ``center``, the grid spanning [-1, 1]^3."""
    x = np.linspace(-1, 1, n, dtype=np.float64)
    return np.sqrt(sum((c - o) ** 2 for c, o in zip(np.meshgrid(x, x, x, indexing="ij"), center)))


def occupancy(n, seed):
    """A float occupancy field in [0, 1]: a smooth ball plus noise."""
    rng = np.random.default_rng(seed)
    return np.clip(1.2 - sphere(n) + 0.15 * rng.standard_normal((n, n, n)), 0, 1).astype(np.float32)


def checker(n):
    i = np.indices((n, n, n)).sum(0)
    return (i % 2).astype(np.uint8)


def specials(seed):
    rng = np.random.default_rng(seed)
    g = rng.uniform(-1, 2, (6, 6, 6)).astype(np.float32)
    flat = g.reshape(-1)
    pick = rng.choice(flat.size, 60, replace=False)
    vals = np.array([0.5, np.nan, np.inf, -np.inf, 3e38, -3e38], np.float32)
    flat[pick] = vals[np.arange(60) % len(vals)]
    return g


SCENES = {
    "cases": (lambda: case_grids(), 0.5),
    "specials": (lambda: np.stack([specials(1), specials(2)]), 0.5),
    "iso_low": (lambda: occupancy(10, 3)[None] - 0.5, -0.2),
    "iso_high": (lambda: occupancy(10, 4)[None], 0.7),
    "views": (lambda: np.stack([(sphere(12) < 0.6).astype(np.float32), occupancy(12, 5),
                                checker(12).astype(np.float32)]), 0.5),
    "checker16": (lambda: checker(16)[None], 0.5),
    "noisy32": (lambda: np.random.default_rng(6).random((1, 32, 32, 32)).astype(np.float32), 0.5),
    "smooth64": (lambda: occupancy(64, 7)[None], 0.5),
}


# Scenes where the reference's operator is wrong but reads only inside its buffers (no face corner of
# the faithful restatement is -3): its dropped voxels at sides 4 and 5, a non-cubic grid and a
# checkerboard past its vertex cap.
QUIRKS = {
    "quirk_n4": (lambda: np.ones((1, 4, 4, 4), np.uint8), 0.5),
    "quirk_n5": (lambda: np.ones((1, 5, 5, 5), np.uint8), 0.5),
    "quirk_noncubic": (lambda: (np.random.default_rng(8).random((1, 6, 9, 7)) < 0.3).astype(np.float32), 0.5),
    "quirk_cap": (lambda: checker(40)[None], 0.5),
}


def same_bits(a, b):
    """Arrays equal bit for bit, NaN taken as one value whatever its payload."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))
