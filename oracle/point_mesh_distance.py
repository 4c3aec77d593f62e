"""TEST INFRASTRUCTURE — an independent float64 point-to-triangle oracle for point_to_mesh_distance.

The closest point of each triangle by Voronoi regions (Ericson, Real-Time Collision Detection, 5.1.5),
written with torch so that it runs on the CPU or the GPU, in float64, chunked over points, and
differentiable by torch autograd.  Regions map to the reference's distance types: 0 the face, 1-3 the
vertices, 4 the edge v1v2, 5 v2v3, 6 v3v1.  It does not follow the reference's arithmetic: it is the
mathematical answer, against which the library's float32 results are held within a stated bound.
"""
import numpy as np
import torch


def _closest(p, a, b, c):
    """p (n, 1, 3), a, b, c (1, F, 3) -> closest points (n, F, 3) and region types (n, F)."""
    ab, ac, ap = b - a, c - a, p - a
    d1, d2 = (ab * ap).sum(-1), (ac * ap).sum(-1)
    bp = p - b
    d3, d4 = (ab * bp).sum(-1), (ac * bp).sum(-1)
    cp = p - c
    d5, d6 = (ab * cp).sum(-1), (ac * cp).sum(-1)
    va = d3 * d6 - d5 * d4
    vb = d5 * d2 - d1 * d6
    vc = d1 * d4 - d3 * d2
    denom = va + vb + vc
    v = vb / denom
    w = vc / denom
    out = a + ab * v[..., None] + ac * w[..., None]
    typ = torch.zeros(out.shape[:-1], dtype=torch.int32, device=p.device)

    def put(mask, point, t):
        nonlocal out, typ
        out = torch.where(mask[..., None], point, out)
        typ = torch.where(mask, torch.full_like(typ, t), typ)

    # later writes take precedence: apply the edges, then the vertices
    e_bc = (va <= 0) & ((d4 - d3) >= 0) & ((d5 - d6) >= 0)
    t_bc = (d4 - d3) / ((d4 - d3) + (d5 - d6))
    put(e_bc, b + (c - b) * t_bc[..., None], 5)
    e_ac = (vb <= 0) & (d2 >= 0) & (d6 <= 0)
    put(e_ac, a + ac * (d2 / (d2 - d6))[..., None], 6)
    e_ab = (vc <= 0) & (d1 >= 0) & (d3 <= 0)
    put(e_ab, a + ab * (d1 / (d1 - d3))[..., None], 4)
    put((d6 >= 0) & (d5 <= d6), c.expand_as(out), 3)
    put((d3 >= 0) & (d4 <= d3), b.expand_as(out), 2)
    put((d1 <= 0) & (d2 <= 0), a.expand_as(out), 1)
    return out, typ


def all_pairs(points, face_vertices):
    """points (N, 3), face_vertices (F, 3, 3) float64 tensors -> (N, F) squared distances and types."""
    p = points[:, None, :]
    a, b, c = (face_vertices[None, :, k, :] for k in range(3))
    q, typ = _closest(p, a, b, c)
    return ((p - q) ** 2).sum(-1), typ


def point_to_mesh_distance(points, face_vertices, chunk_pairs=1 << 24):
    """points (N, 3), face_vertices (F, 3, 3) (numpy or torch; computed in float64 on their device) ->
    (dist (N,), face (N,) int64, type (N,) int32, min distance of every face (N, F) not kept)."""
    p = torch.as_tensor(points).to(torch.float64)
    fv = torch.as_tensor(face_vertices).to(torch.float64).to(p.device)
    n, f = p.shape[0], fv.shape[0]
    step = max(1, chunk_pairs // max(f, 1))
    dist, face, typ = [], [], []
    for s in range(0, n, step):
        d, t = all_pairs(p[s:s + step], fv)
        m, i = d.min(1)
        dist.append(m)
        face.append(i)
        typ.append(t.gather(1, i[:, None])[:, 0])
    return torch.cat(dist), torch.cat(face), torch.cat(typ)


def distance_to_faces(points, face_vertices, face):
    """The float64 squared distance of each point to its given face (differentiable)."""
    fv = face_vertices[face]
    q, _ = _closest(points[:, None, :], fv[:, None, 0], fv[:, None, 1], fv[:, None, 2])
    q = q[:, 0]
    return ((points - q) ** 2).sum(-1)


def numpy_distance(points, face_vertices):
    """Convenience: numpy in, numpy out (dist, face, type)."""
    d, f, t = point_to_mesh_distance(np.asarray(points, np.float64), np.asarray(face_vertices, np.float64))
    return d.numpy(), f.numpy(), t.numpy()
