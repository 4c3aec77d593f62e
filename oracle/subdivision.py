"""Torch restatement of Loop subdivision (kaolin/ops/mesh/trianglemesh.py:482-612,
subdivide_trianglemesh) for any batch, in float32 or float64, with autograd to the vertices and alpha.

Per level, with V vertices and F faces:
  edges    the sorted face edges (f0,f1), (f1,f2), (f2,f0), made unique in lexicographic order (E of
           them, each with its count of face edges); edge e becomes vertex V + e
  n        the number of unique neighbours of each vertex, a self-loop counted once
  alpha    given (B, V), or Loop's weight computed in float32 as the reference does (NaN for n = 0)
  even     (1 - a_i) x_i + (a_i / n_i) sum_{j in N(i)} x_j
  odd      an edge of two face edges: (both faces' vertices + both endpoints) / 8; else the midpoint;
           the next level's alpha: the old alpha for even rows, the same stencils over alpha for odd rows
  faces    (v0, v1, v2, V+e01, V+e12, V+e20)[[1,4,3], [0,3,5], [2,5,4], [5,3,4]] for each face in order
The structures are built with numpy; the arithmetic is torch, in the dtype of the vertices.
"""
import math

import numpy as np
import torch

CHILDREN = np.array([[1, 4, 3], [0, 3, 5], [2, 5, 4], [5, 3, 4]])


def level(num_vertices, faces):
    """-> dict of the level's structures: edges (E, 2), two-face edges and their faces, degree, pairs."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    V, F = int(num_vertices), len(faces)
    if F and (faces.min() < 0 or faces.max() >= V):
        raise IndexError("face index outside [0, V)")
    fe = np.sort(np.stack([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]], 1).reshape(-1, 2), 1)
    key = fe[:, 0] * max(V, 1) + fe[:, 1]
    uniq, inverse, counts = np.unique(key, return_inverse=True, return_counts=True)
    inverse = inverse.reshape(-1)
    edges = np.stack([uniq // max(V, 1), uniq % max(V, 1)], 1).astype(np.int64)
    two = np.nonzero(counts == 2)[0]
    # the faces of each two-face edge: its face edges sorted by (edge, face-edge index)
    q = np.nonzero(counts[inverse] == 2)[0]
    q = q[np.lexsort((q, inverse[q]))]
    two_faces = (q // 3).reshape(-1, 2)
    pairs = np.unique(np.concatenate([edges, edges[:, ::-1]]), axis=0) if F else np.zeros((0, 2), np.int64)
    degree = np.bincount(pairs[:, 0], minlength=V)
    table = np.concatenate([faces, inverse.reshape(F, 3) + V], 1)
    new_faces = table[:, CHILDREN].reshape(-1, 3)
    return dict(V=V, F=F, faces=faces, edges=edges, two=two, two_faces=two_faces, other=np.nonzero(counts != 2)[0],
                pairs=pairs, degree=degree, new_faces=new_faces)


def default_alpha(degree):
    """The reference's _get_alpha(n) * n, in float32 with torch's own steps (2*pi / n = reciprocal(n) * 2*pi)."""
    n = torch.as_tensor(degree).float()
    c = 0.375 + 0.25 * torch.cos(torch.reciprocal(n) * (2 * math.pi))
    a = (0.625 - c * c) / n
    a[n == 3] = 3 / 16
    return a * n


def stencil(t, lv):
    """The odd rows over t (B, V, C): two-face edges (8 values) / 8, the others (a + b) / 2."""
    B, C = t.shape[0], t.shape[-1]
    out = t.new_zeros((B, len(lv["edges"]), C))
    e = lv["edges"]
    dev = t.device
    other, two = torch.from_numpy(lv["other"]).to(dev), torch.from_numpy(lv["two"]).to(dev)
    out[:, other] = (t[:, e[lv["other"], 0]] + t[:, e[lv["other"], 1]]) / 2
    if len(lv["two"]):
        idx = np.concatenate([lv["faces"][lv["two_faces"]].reshape(-1, 6), e[lv["two"]]], 1)      # (E2, 8)
        out[:, two] = t[:, torch.from_numpy(idx).to(dev)].sum(2) / 8
    return out


def apply_level(lv, x, alpha=None):
    """One level: x (B, V, 3), alpha (B, V) or None -> (y (B, V + E, 3), next alpha (B, V + E) or None)."""
    dev = x.device
    n = torch.from_numpy(lv["degree"]).to(dev, x.dtype)
    a = default_alpha(lv["degree"]).to(dev, x.dtype)[None] if alpha is None else alpha
    rows, cols = (torch.from_numpy(lv["pairs"][:, k]).to(dev) for k in (0, 1))
    s = x.new_zeros(x.shape).index_add(1, rows, x[:, cols])
    even = (1 - a)[..., None] * x + (a / n)[..., None] * s
    y = torch.cat([even, stencil(x, lv)], 1)
    if alpha is None:
        return y, None
    return y, torch.cat([alpha, stencil(alpha[..., None], lv)[..., 0]], 1)


def subdivide(vertices, faces, iterations, alpha=None):
    """subdivide_trianglemesh for vertices (B, V, 3) of any batch and dtype, faces (F, 3) -> (vertices, faces)."""
    x, f = vertices, np.asarray(faces, np.int64).reshape(-1, 3)
    for _ in range(int(iterations)):
        lv = level(x.shape[1], f)
        x, alpha = apply_level(lv, x, alpha)
        f = lv["new_faces"]
    return x, torch.from_numpy(np.ascontiguousarray(f))
