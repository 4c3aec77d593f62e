"""TEST INFRASTRUCTURE — NOT PRODUCT CODE.

ctypes front-end of oracle/check_sign.c, the brute-force CPU restatement of the reference's point-in-mesh
test (``kaolin.ops.mesh.check_sign`` and its operator ``unbatched_mesh_intersection_cuda``), in float32
and float64.  ``build()`` compiles it with gcc -ffp-contract=off into oracle/_build/ (called from
``__graft_entry__.build()``).
"""
import ctypes
import functools
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "check_sign.c")
_LIB = os.path.join(_HERE, "_build", "libcheck_sign_oracle.so")
FIXTURE = os.path.join(os.path.dirname(_HERE), "tests", "golden", "check_sign.npz")   # the reference test's
_lib = None
_SFX = {np.dtype(np.float32): "f32", np.dtype(np.float64): "f64"}


def build(force=False):
    """gcc -O2 -fopenmp -ffp-contract=off (no compiler-added FMA fusion)."""
    if not force and os.path.exists(_LIB) and os.path.getmtime(_LIB) >= os.path.getmtime(_SRC):
        return _LIB
    os.makedirs(os.path.dirname(_LIB), exist_ok=True)
    subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off",
                           "-fno-fast-math", "-o", _LIB, _SRC, "-lm"])
    return _LIB


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_LIB)
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def mesh_intersection_count(points, verts_1, verts_2, verts_3):
    """unbatched_mesh_intersection_cuda: points (N, 3), corners (F, 3) of one float dtype -> counts (N,)."""
    dt = np.asarray(points).dtype
    pts, v1, v2, v3 = (np.ascontiguousarray(a, dtype=dt) for a in (points, verts_1, verts_2, verts_3))
    out = np.zeros(pts.shape[0], dtype=dt)
    fn = getattr(lib(), "oracle_mesh_intersection_count_" + _SFX[dt])
    fn(ctypes.c_int(pts.shape[0]), _p(pts), ctypes.c_int(v1.shape[0]), _p(v1), _p(v2), _p(v3), _p(out))
    return out


def check_sign(verts, faces, points):
    """check_sign's CUDA path: verts (B, V, 3), faces (F, 3) int64, points (B, N, 3) -> (B, N) bool.
    Raises IndexError for a face index outside [0, V)."""
    dt = np.asarray(verts).dtype
    v = np.ascontiguousarray(verts, dtype=dt)
    f = np.ascontiguousarray(faces, dtype=np.int64)
    q = np.ascontiguousarray(points, dtype=dt)
    B, V, _ = v.shape
    F, N = f.shape[0], q.shape[1]
    out = np.zeros((B, N), dtype=np.uint8)
    scratch = np.empty(9 * F + 4 * N + 1, dtype=dt)
    fn = getattr(lib(), "oracle_check_sign_" + _SFX[dt])
    if fn(ctypes.c_int(B), ctypes.c_int(V), ctypes.c_int(F), ctypes.c_int(N), _p(v), _p(f), _p(q), _p(scratch),
          _p(out)) != 0:
        raise IndexError("faces holds an index outside [0, V)")
    return out.astype(bool)


# ---- constructed scenes, shared by the CPU and GPU tests and the stored reference outputs ----
# Every scene is float64 data; a float32 case rounds it.  check_sign scenes: verts (B, V, 3), faces (F, 3),
# points (B, N, 3); raw-operator scenes (name "raw_*"): points (N, 3), verts_1, verts_2, verts_3 (F, 3).

CAP = 16                    # kMaxCells of kaolin_b200/csrc/grid_bins.cuh


def grid_side(F):
    G = 8
    while G < 256 and G * G < F:
        G += 8
    return G


def _box_lattice(n, size=4.0):
    """The closed surface of the cube [0, size]^3, each side an n x n lattice of squares split along
    one diagonal: (V, 3), (12 n^2, 3)."""
    t = np.linspace(0.0, size, n + 1)
    verts, faces = [], []
    for axis in range(3):
        for side in (0.0, size):
            u, w = np.meshgrid(t, t, indexing="ij")
            p = np.zeros((n + 1, n + 1, 3))
            p[..., axis], p[..., (axis + 1) % 3], p[..., (axis + 2) % 3] = side, u, w
            base = sum(len(v) for v in verts)
            verts.append(p.reshape(-1, 3))
            idx = base + np.arange((n + 1) ** 2).reshape(n + 1, n + 1)
            a, b, c, d = idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]
            tri = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([a, c, d], -1).reshape(-1, 3)])
            faces.append(tri if side else tri[:, ::-1])
    v = np.concatenate(verts)
    uniq, inv = np.unique(v, axis=0, return_inverse=True)
    return uniq, inv.reshape(-1)[np.concatenate(faces)]


def _icosphere(level, rng=None, noise=0.0):
    from kaolin_b200 import synthetic
    v, f = synthetic.icosphere(level)
    if rng is not None and noise:
        v = v * (1.0 + noise * rng.uniform(-1, 1, size=(v.shape[0], 1)))
    return v, f


def _soup(rng, F, size):
    """F random triangles of edge ~size in the unit cube."""
    c = rng.uniform(0.0, 1.0, size=(F, 1, 3))
    tri = c + size * rng.normal(size=(F, 3, 3))
    return tri.reshape(-1, 3), np.arange(3 * F, dtype=np.int64).reshape(F, 3)


def _uniform(rng, verts, n, margin=0.1):
    lo, hi = verts.min(0), verts.max(0)
    pad = margin * (hi - lo)
    return rng.uniform(lo - pad, hi + pad, size=(n, 3))


def _lattice_points(n, size, xs, offsets):
    """Points whose (y, z) sit on the side lattice of _box_lattice(n, size), shifted by `offsets` (in
    lattice steps), at each x of `xs`."""
    h = size / n
    k = np.arange(n + 1) * h
    out = []
    for dy, dz in offsets:
        y, z = np.meshgrid(k + dy * h, k + dz * h, indexing="ij")
        for x in xs:
            out.append(np.stack([np.full(y.size, x), y.reshape(-1), z.reshape(-1)], -1))
    return np.concatenate(out)


def _cap_faces(G, size):
    """Faces inside the cube whose y-z boxes, in cells of a G x G grid over [0, size], are 4 x 4 (the
    cap, bounds on cell borders), 1 x 16, 1 x 17, 3 x 6 and 4 x 5, at x = size / 2 and x = size / 3."""
    h = size / G
    faces = []
    for x in (size / 2, size / 3):
        for (ny, nz), (y0, z0) in (((4, 4), (3, 5)), ((1, 16), (10, 2)), ((1, 17), (20, 1)), ((3, 6), (7, 20)),
                                   ((4, 5), (14, 14)), ((16, 1), (2, 27)), ((17, 1), (5, 30))):
            # bounds on borders: the upper bound's border opens the next cell, so span n - 1 steps
            y1, z1 = y0 + ny - 1, z0 + nz - 1
            faces.append([[x, y0 * h, z0 * h], [x + h, y1 * h, z0 * h], [x, y0 * h, z1 * h]])
            faces.append([[x, y1 * h, z1 * h], [x - h, y0 * h, z1 * h], [x, y1 * h, z0 * h]])
    return np.array(faces)


@functools.lru_cache(maxsize=1)
def scenes():
    """name -> dict of float64 arrays (see above)."""
    rng = np.random.default_rng(20261017)
    out = {}
    with np.load(FIXTURE) as z:
        fx = {k: z[k] for k in z.files}
    out["fixture"] = dict(verts=fx["verts"], faces=fx["faces"], points=fx["points"])
    out["fixture_zero_area"] = dict(verts=fx["verts"], faces=np.concatenate([fx["faces"], fx["zero_area_faces"]]),
                                    points=fx["points"])

    # shared vertices and edges of a lattice: on-vertex, on-edge of constant y (the vertical-edge rule),
    # of constant z and on the diagonals, at x outside, on and inside the cube; n = 8 gives G = 32, so
    # every lattice line is also a cell border
    v, f = _box_lattice(8)
    offs = [(0, 0), (0.5, 0), (0, 0.5), (0.5, 0.5), (0.25, 0.25), (0.25, 0.75)]
    p = _lattice_points(8, 4.0, [-1.0, 0.0, 1.25, 2.0, 4.0, 5.5], offs)
    out["lattice"] = dict(verts=v[None], faces=f, points=p[None])
    v3, f3 = _box_lattice(6, 3.0)          # maxlen 3: normalised lattice coordinates are inexact
    p3 = _lattice_points(6, 3.0, [-0.5, 1.0, 2.5, 3.5], offs)
    out["lattice_inexact"] = dict(verts=v3[None], faces=f3, points=p3[None])
    vi, fi = _icosphere(3)
    rot = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    vi = vi @ rot.T
    e = np.concatenate([fi[:, [0, 1]], fi[:, [1, 2]], fi[:, [2, 0]]])
    mids = (vi[e[:, 0]] + vi[e[:, 1]]) / 2
    yz = np.concatenate([vi[:, 1:], mids[:, 1:]])
    p = np.concatenate([np.concatenate([np.full((len(yz), 1), x), yz], 1) for x in (-2.0, 0.0, 0.3, 2.0)])
    out["icosphere_vertices_edges"] = dict(verts=vi[None], faces=fi, points=p[None])

    # cell borders and the cap: the lattice plus faces of exactly 16 cells and more
    cf = _cap_faces(32, 4.0)
    vc = np.concatenate([v, cf.reshape(-1, 3)])
    fc = np.concatenate([f, len(v) + np.arange(cf.shape[0] * 3).reshape(-1, 3)])
    pc = np.concatenate([_lattice_points(32, 4.0, [0.1, 1.9, 3.0], [(0, 0), (0.5, 0)]),
                         _uniform(rng, v, 3000, 0.0)])
    out["cell_borders_cap"] = dict(verts=vc[None], faces=fc, points=pc[None])
    vw, fw = [], []
    while len(fw) < 40:                    # big triangles only: every face on the wide list
        t = rng.uniform(0, 1, size=(3, 3))
        if np.ptp(t[:, 1]) > 0.6 and np.ptp(t[:, 2]) > 0.6:
            fw.append(np.arange(3) + 3 * len(fw)); vw.append(t)
    vw = np.concatenate(vw)
    out["wide_only"] = dict(verts=vw[None], faces=np.array(fw), points=_uniform(rng, vw, 3000)[None])

    # G across its range
    for F, size in ((30, 0.3), (3000, 0.05), (17000, 0.02), (70000, 0.01)):
        vs, fs = _soup(rng, F, size)
        out[f"soup_G{grid_side(F)}"] = dict(verts=vs[None], faces=fs, points=_uniform(rng, vs, 3000)[None])

    # B = 3, different vertices per view
    vb = np.stack([_icosphere(3, rng, 0.1)[0] * s + o for s, o in ((1.0, 0.0), (2.5, 1.0), (0.5, -3.0))])
    pb = np.stack([_uniform(rng, x, 2000) for x in vb])
    out["batch3"] = dict(verts=vb, faces=_icosphere(3)[1], points=pb)

    # degenerate input
    v2, f2 = _icosphere(2)
    base = _uniform(rng, v2, 600)
    special = np.array([np.nan, np.inf, -np.inf, 1e30, -1e30, 3e38, 0.0])
    odd = np.array([[a, b, c] for a in special for b in special[[0, 1, 2, 3, 6]] for c in special[[0, 1, 2, 4, 6]]])
    out["nan_inf_points"] = dict(verts=v2[None], faces=f2, points=np.concatenate([base, odd])[None])
    for name, extra in (("nan_vertex", [np.nan, 0, 0]), ("inf_vertex", [np.inf, 0, 0]), ("far_vertex", [1e6, 0, 0])):
        out[name] = dict(verts=np.concatenate([v2, [extra]])[None], faces=f2, points=base[None])
    out["zero_maxlen"] = dict(verts=np.full((1, 12, 3), 0.5), faces=f2[:20] % 12,
                              points=np.concatenate([base[:100], np.full((3, 3), 0.5), np.zeros((2, 3))])[None])
    dup = np.concatenate([f2, f2[::3], f2[::7], f2[::7]])
    out["duplicate_faces"] = dict(verts=v2[None], faces=dup, points=base[None])
    far = np.concatenate([base[:200], rng.uniform(-1, 1, size=(200, 3)) * np.array([1e30, 1e3, 1e3]),
                          rng.uniform(-1, 1, size=(200, 3)) * np.array([1, 1e20, 1e20])])
    out["far_points"] = dict(verts=v2[None], faces=f2, points=far[None])

    # the raw operator: corners as given, NaN and infinities in them
    vs, fs = _soup(rng, 2000, 0.1)
    tri = vs[fs]
    out["raw_soup"] = dict(points=_uniform(rng, vs, 4000), verts_1=tri[:, 0], verts_2=tri[:, 1], verts_3=tri[:, 2])
    tri = vs[fs][:600].copy()
    tri[0:50, 0, 1] = np.nan                       # one corner's y NaN: the box skips it
    tri[50:100, :, 1] = np.nan                     # the whole y box NaN: dropped by the binning
    tri[100:150, :, 2] = np.nan
    tri[150:200, 1, 0] = np.nan
    tri[200:250, 2, 2] = np.inf
    tri[250:300, 0, 1] = -np.inf
    tri[300:350, :, 0] = np.inf
    pts = np.concatenate([_uniform(rng, vs, 2000), odd])
    out["raw_nan_inf"] = dict(points=pts, verts_1=tri[:, 0], verts_2=tri[:, 1], verts_3=tri[:, 2])
    return out


def is_raw(scene):
    return "verts_1" in scene


def cast(scene, dtype):
    return {k: (a if a.dtype == np.int64 else a.astype(dtype)) for k, a in scene.items()}


def oracle_counts(scene):
    """The C oracle's counts for a scene: (B, N) (check_sign, before the parity) or (N,) (raw)."""
    if is_raw(scene):
        return mesh_intersection_count(scene["points"], scene["verts_1"], scene["verts_2"], scene["verts_3"])
    v, f, q = scene["verts"], scene["faces"], scene["points"]
    dt = v.dtype
    out = []
    with np.errstate(all="ignore"):
        for b in range(v.shape[0]):
            lens = [v[b, :, a].max() - v[b, :, a].min() for a in range(3)]   # np.max propagates NaN
            m = np.array(lens, dtype=dt).max()
            vb, qb = (v[b] / m).astype(dt), (q[b] / m).astype(dt)
            out.append(mesh_intersection_count(qb, vb[f[:, 0]], vb[f[:, 1]], vb[f[:, 2]]))
    return np.stack(out)


def binning(scene):
    """Host restatement of check_sign.cu's binning of each view, in float32 as the kernels compute it:
    G, the face cell counts (0 for a dropped NaN box), and the points' cell coordinates (y, z) before
    the clamp.  Needs the normalised corners, so it normalises as oracle_counts does."""
    f32 = np.float32
    if is_raw(scene):
        views = [(np.stack([scene["verts_1"], scene["verts_2"], scene["verts_3"]], 1), scene["points"])]
    else:
        v, f, q = scene["verts"], scene["faces"], scene["points"]
        views = []
        with np.errstate(all="ignore"):
            for b in range(v.shape[0]):
                m = np.array([v[b, :, a].max() - v[b, :, a].min() for a in range(3)], dtype=v.dtype).max()
                views.append((((v[b] / m).astype(v.dtype))[f], (q[b] / m).astype(v.dtype)))
    out = []
    with np.errstate(all="ignore"):
        for tri, pts in views:
            F = tri.shape[0]
            G = grid_side(F)
            lo = np.fmin.reduce(tri[:, :, 1:], axis=1).astype(f32)
            hi = np.fmax.reduce(tri[:, :, 1:], axis=1).astype(f32)
            bounds = []
            for k in range(2):
                a = np.fmin.reduce(lo[:, k], initial=np.inf)
                z = np.fmax.reduce(hi[:, k], initial=-np.inf)
                if not (z >= a) or not (f32(z - a) < np.inf):
                    a, z = f32(0), f32(1)
                bounds.append((f32(a), f32(f32(G) / np.fmax(f32(z - a), f32(1e-20)))))
            coord = lambda x, k: f32(np.asarray(x, f32) - bounds[k][0]) * bounds[k][1]
            cell = lambda x, k: np.fmin(np.fmax(coord(x, k), f32(0)), f32(G - 1)).astype(np.int64)
            ok = (hi[:, 0] >= lo[:, 0]) & (hi[:, 1] >= lo[:, 1])
            ncell = np.where(ok, (cell(hi[:, 0], 0) - cell(lo[:, 0], 0) + 1) * (cell(hi[:, 1], 1) - cell(lo[:, 1], 1) + 1), 0)
            out.append(dict(G=G, ncell=ncell, box_coord=(coord(lo[:, 0], 0), coord(lo[:, 1], 1)),
                            point_coord=(coord(pts[:, 1], 0), coord(pts[:, 2], 1))))
    return out
