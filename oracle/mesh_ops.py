"""Numpy restatement of the mesh topology, uniform Laplacian and vertex averaging
(kaolin/ops/mesh/mesh.py:78-208, kaolin/metrics/trianglemesh.py:318-350) in the terms of
kaolin_b200/csrc/mesh_topology.cu: the corner and adjacency CSRs, the Laplacian applied in fp64 with
the fp32 weights fl(1 / degree) widened to fp64, and the averaging summed in fp32 in key order."""
import numpy as np


def topology(num_vertices, faces):
    """-> dict of corner_ptr (V+1), corners (F*S, corner ids f*S + k in key order k*F + f), adj_ptr (V+1),
    adj (E) ascending per row, degree (V), weight (V) float32."""
    faces = np.asarray(faces, dtype=np.int64)
    V = int(num_vertices)
    F, S = faces.shape
    if F and (faces.min() < 0 or faces.max() >= V):
        raise IndexError("face index outside [0, V)")
    f, k = np.meshgrid(np.arange(F), np.arange(S), indexing="ij")
    vert = faces.reshape(-1)
    key = (k * F + f).reshape(-1)
    order = np.lexsort((key, vert))                       # by vertex, then key
    corners = (f * S + k).reshape(-1)[order]
    corner_ptr = np.zeros(V + 1, np.int64)
    np.add.at(corner_ptr, vert + 1, 1)
    corner_ptr = np.cumsum(corner_ptr)
    nxt = np.roll(faces, -1, axis=1).reshape(-1)
    prv = np.roll(faces, 1, axis=1).reshape(-1)
    pairs = np.unique(np.stack([np.concatenate([vert, vert]), np.concatenate([nxt, prv])], 1), axis=0) \
        if F else np.zeros((0, 2), np.int64)
    degree = np.bincount(pairs[:, 0], minlength=V).astype(np.int64)
    adj_ptr = np.concatenate([[0], np.cumsum(degree)])
    with np.errstate(divide="ignore"):
        weight = np.where(degree > 0, np.float32(1) / np.maximum(degree, 1).astype(np.float32), 0).astype(np.float32)
    return dict(corner_ptr=corner_ptr, corners=corners, adj_ptr=adj_ptr, adj=pairs[:, 1].copy(), rows=pairs[:, 0].copy(),
                degree=degree, weight=weight, V=V, faces=faces)


def dense_laplacian(t):
    V = t["V"]
    L = np.zeros((V, V), np.float32)
    L[t["rows"], t["adj"]] = t["weight"][t["rows"]]
    L[np.arange(V), np.arange(V)] = -1
    return L


def dense_adjacency(t):
    A = np.zeros((t["V"], t["V"]), np.float32)
    A[t["rows"], t["adj"]] = 1
    return A


def apply(t, x, transpose=False, smooth=False):
    """(L or L^T, + I if smooth) x in fp64 for x (V, C) or (B, V, C); the off-diagonal weights are fl(1/deg)."""
    x = np.asarray(x, np.float64)
    xb = x.reshape((-1,) + x.shape[-2:])
    off = t["rows"] != t["adj"]
    r, c = t["rows"][off], t["adj"][off]
    w = t["weight"].astype(np.float64)[r]
    src, dst = (r, c) if transpose else (c, r)       # L x: y_i += w_i x_j;  L^T x: y_j += w_i x_i
    y = np.zeros_like(xb)
    for b in range(len(xb)):
        np.add.at(y[b], dst, w[:, None] * xb[b][src])
    y = y.reshape(x.shape)
    return y if smooth else y - x


def average(t, face_features):
    """average_face_vertex_features in fp32, summed in key order, divided by max(count, 1)."""
    ff = np.asarray(face_features, np.float32)
    B, F, S, N = ff.shape
    V = t["V"]
    flat = ff.reshape(B, F * S, N)
    cp, corners = t["corner_ptr"], t["corners"]
    counts = np.diff(cp)
    s = np.zeros((B, V, N), np.float32)
    for p in range(int(counts.max()) if V else 0):      # the p-th corner of every row, in key order
        rows = np.nonzero(counts > p)[0]
        s[:, rows] = s[:, rows] + flat[:, corners[cp[rows] + p]]
    return s / np.maximum(counts, 1).astype(np.float32)[None, :, None]


def average_backward(t, grad_out, num_faces, face_size):
    g = np.asarray(grad_out, np.float32)
    counts = np.maximum(np.diff(t["corner_ptr"]), 1).astype(np.float32)
    fl = t["faces"].reshape(-1)
    return (g[:, fl] / counts[fl][None, :, None]).reshape(g.shape[0], num_faces, face_size, g.shape[-1])
