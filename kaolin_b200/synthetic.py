"""Synthetic scenes for the parity tests and bench.py (SURVEY.md §8d).

G1 ``icosphere_views``: a closed, outward-oriented icosphere (20*4^L faces) with
per-mesh radial jitter and a random rotation, seen by a perspective camera
(fov 45 deg) from a radius-3 sphere looking at the origin — the same geometry
the reference's test fixtures use (tests/python/kaolin/render/mesh/
test_rasterization.py:52-75; camera maths as kaolin/render/camera/legacy.py).
G2 ``triangle_soup``: independent random triangles.

All outputs are float32 numpy arrays in the layout of
``kaolin.render.mesh.dibr_rasterization``'s arguments:
face_vertices_z (B,F,3), face_vertices_image (B,F,3,2) in [-1,1],
face_normals_z (B,F).
"""
import math

import numpy as np

_T = (1.0 + math.sqrt(5.0)) / 2.0
_ICO_V = np.array([[-1, _T, 0], [1, _T, 0], [-1, -_T, 0], [1, -_T, 0],
                   [0, -1, _T], [0, 1, _T], [0, -1, -_T], [0, 1, -_T],
                   [_T, 0, -1], [_T, 0, 1], [-_T, 0, -1], [-_T, 0, 1]], dtype=np.float64)
_ICO_F = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11],
                   [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6], [7, 1, 8],
                   [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9],
                   [4, 9, 5], [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]], dtype=np.int64)
_CACHE = {}


def icosphere(level):
    """Unit icosphere: (V,3) float64 vertices, (20*4^level, 3) int64 faces (outward CCW)."""
    if level in _CACHE:
        return _CACHE[level]
    v = _ICO_V / np.linalg.norm(_ICO_V, axis=1, keepdims=True)
    f = _ICO_F
    for _ in range(level):
        e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]], 0)
        key = np.sort(e, 1)
        uniq, inv = np.unique(key, axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        mid = v[uniq[:, 0]] + v[uniq[:, 1]]
        mid /= np.linalg.norm(mid, axis=1, keepdims=True)
        n0 = v.shape[0]
        v = np.concatenate([v, mid], 0)
        nf = f.shape[0]
        ab, bc, ca = n0 + inv[:nf], n0 + inv[nf:2 * nf], n0 + inv[2 * nf:]
        a, b, c = f[:, 0], f[:, 1], f[:, 2]
        f = np.concatenate([np.stack([a, ab, ca], 1), np.stack([b, bc, ab], 1),
                            np.stack([c, ca, bc], 1), np.stack([ab, bc, ca], 1)], 0)
    _CACHE[level] = (v, f)
    return v, f


def _random_rotation(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _look_at(eye):
    """World->camera rotation rows (right, up, backward) for a camera at `eye` looking at 0."""
    back = eye / np.linalg.norm(eye)
    up = np.array([0.0, 1.0, 0.0])
    if abs(back @ up) > 0.999:
        up = np.array([1.0, 0.0, 0.0])
    right = np.cross(up, back)
    right /= np.linalg.norm(right)
    upv = np.cross(back, right)
    return np.stack([right, upv, back], 0)


def project_mesh(vertices, faces, eye, fov=math.pi / 4.0):
    """vertices (V,3) world -> (fvz (F,3), fvi (F,3,2), fnz (F,)) float32."""
    R = _look_at(np.asarray(eye, dtype=np.float64))
    vc = (vertices - eye) @ R.T                     # camera space, looking down -z
    t = math.tan(fov / 2.0)
    img = vc[:, :2] / (-vc[:, 2:3] * t)
    fv = vc[faces]                                   # (F,3,3)
    n = np.cross(fv[:, 1] - fv[:, 0], fv[:, 2] - fv[:, 0])
    n /= np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-20)
    return (fv[..., 2].astype(np.float32), img[faces].astype(np.float32),
            n[:, 2].astype(np.float32))


def icosphere_views(batch, level, seed=0, jitter=0.05, same_mesh=False, radius=3.0):
    """G1: `batch` views; a differently jittered/rotated mesh per view unless same_mesh."""
    rng = np.random.default_rng(seed)
    v0, f = icosphere(level)
    fvz = np.empty((batch, f.shape[0], 3), np.float32)
    fvi = np.empty((batch, f.shape[0], 3, 2), np.float32)
    fnz = np.empty((batch, f.shape[0]), np.float32)
    v = None
    for b in range(batch):
        if v is None or not same_mesh:
            r = 1.0 + jitter * rng.uniform(-1, 1, size=(v0.shape[0], 1))
            v = (v0 * r) @ _random_rotation(rng).T
        d = rng.normal(size=3)
        eye = radius * d / np.linalg.norm(d)
        fvz[b], fvi[b], fnz[b] = project_mesh(v, f, eye)
    return fvz, fvi, fnz


def triangle_soup(batch, num_faces, seed=0, coverage=1.5):
    """G2: random triangles; centres U(-0.9,0.9)^2, vertex offsets N(0, s^2)."""
    rng = np.random.default_rng(seed)
    s = math.sqrt(coverage * 4.0 / num_faces) / 2.0
    c = rng.uniform(-0.9, 0.9, size=(batch, num_faces, 1, 2))
    fvi = (c + rng.normal(scale=s, size=(batch, num_faces, 3, 2))).astype(np.float32)
    fvz = rng.uniform(-3.0, -1.0, size=(batch, num_faces, 3)).astype(np.float32)
    fnz = np.where(rng.uniform(size=(batch, num_faces)) < 0.75, 1.0, -1.0).astype(np.float32)
    return fvz, fvi, fnz


def freudenthal_grid(res):
    """A tet grid over [-0.5, 0.5]^3: (res + 1)^3 vertices (V, 3) float32 and 6 res^3 tets (T, 4)
    int64, each cube cell split into six tets around its diagonal (0,0,0)-(1,1,1) (the Freudenthal,
    or Kuhn, triangulation), so neighbouring cells share their faces' diagonals."""
    n = res + 1
    g = np.arange(n, dtype=np.float64) / res - 0.5
    verts = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    i, j, k = (a.reshape(-1) for a in np.meshgrid(*(np.arange(res),) * 3, indexing="ij"))
    idx = lambda a, b, c: ((i + a) * n + (j + b)) * n + (k + c)
    unit = np.eye(3, dtype=np.int64)
    tets = []
    for p in ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)):
        c1 = unit[p[0]]
        c2 = c1 + unit[p[1]]
        tets.append(np.stack([idx(0, 0, 0), idx(*c1), idx(*c2), idx(1, 1, 1)], 1))
    return verts, np.stack(tets, 1).reshape(-1, 4).astype(np.int64)


def random_features(batch, num_faces, dim, seed=0):
    rng = np.random.default_rng(seed + 7919)
    return rng.uniform(size=(batch, num_faces, 3, dim)).astype(np.float32)
