"""Writes tests/golden/mesh_ops.npz from the reference's own adjacency_matrix, uniform_laplacian,
average_face_vertex_features, compute_vertex_normals and uniform_laplacian_smoothing, run on the CPU
(imported in place through oracle/ref_import; the pure-torch modules need no extension).

Per case <c>: faces, V, and for each function its output; for smoothing (B, V, 3) vertices, the output
and the gradient of sum(out * w); for averaging (B, F, S, N) features, the output and the gradient of
sum(out * w); and the sparse adjacency's indices and values.

    python tests/golden/make_mesh_ops_golden.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, ROOT)

from oracle import ref_import  # noqa: E402
from kaolin_b200 import synthetic  # noqa: E402


def random_mesh(rng, V, F, S):
    """Random faces over V vertices with degenerate faces, duplicate faces and unreferenced vertices."""
    used = rng.permutation(V)[: V - 3]                 # three vertices referenced by no face
    faces = rng.choice(used, size=(F, S))
    faces[1, 1] = faces[1, 0]                          # degenerate: a repeated vertex
    faces[2, :] = faces[2, 0]                          # fully degenerate: a self-loop only
    faces[3] = faces[4]                                # duplicate face
    faces[5] = np.roll(faces[6], 1)                    # the same face, rotated
    return faces


def cases():
    rng = np.random.default_rng(1234)
    out = {
        "ref_adjacency": (5, np.array([[1, 3, 2], [1, 4, 0]])),
        "ref_average": (7, np.array([[0, 1, 2], [1, 2, 4], [2, 4, 5], [2, 5, 6]])),
        "ref_normals": (6, np.array([[0, 2, 1], [0, 3, 2], [0, 4, 3]])),
        "ref_smooth": (3, np.array([[0, 1, 2]])),
        "tri": (64, random_mesh(rng, 64, 120, 3)),
        "quad": (48, random_mesh(rng, 48, 60, 4)),
        "pent": (30, random_mesh(rng, 30, 25, 5)),
        "empty": (4, np.zeros((0, 3), np.int64)),
    }
    v, f = synthetic.icosphere(3)
    out["ico3"] = (len(v), np.asarray(f))
    return out


def main():
    mm = ref_import.module("kaolin.ops.mesh.mesh")
    tm = ref_import.module("kaolin.metrics.trianglemesh")
    rng = np.random.default_rng(5)
    g = {}
    for name, (V, faces) in cases().items():
        faces_t = torch.from_numpy(np.asarray(faces, np.int64))
        F, S = faces_t.shape
        g[f"{name}_faces"] = faces_t.numpy()
        g[f"{name}_V"] = np.int64(V)
        g[f"{name}_laplacian"] = mm.uniform_laplacian(V, faces_t).numpy()
        g[f"{name}_adjacency_dense"] = mm.adjacency_matrix(V, faces_t, sparse=False).numpy()
        sp = mm.adjacency_matrix(V, faces_t)
        g[f"{name}_adjacency_indices"] = sp._indices().numpy()
        g[f"{name}_adjacency_values"] = sp._values().numpy()

        B = 2
        verts = torch.from_numpy(rng.normal(size=(B, V, 3)).astype(np.float32)).requires_grad_(True)
        if name == "ref_smooth":
            verts = torch.tensor([[[0, 0, 1], [2, 1, 2], [3, 1, 2]], [[3, 1, 2], [0, 0, 3], [0, 3, 3]]],
                                 dtype=torch.float32, requires_grad=True)
        w = torch.from_numpy(rng.normal(size=(B, V, 3)).astype(np.float32))
        smooth = tm.uniform_laplacian_smoothing(verts, faces_t)
        (smooth * w).sum().backward()
        g[f"{name}_smooth_vertices"] = verts.detach().numpy()
        g[f"{name}_smooth_w"] = w.numpy()
        g[f"{name}_smooth"] = smooth.detach().numpy()
        g[f"{name}_smooth_grad"] = verts.grad.numpy()

        N = 10 if name == "ref_average" else 3
        ff = torch.from_numpy((rng.normal(size=(3, F, S, N)) * 100).astype(np.float32)).requires_grad_(True)
        avg = mm.average_face_vertex_features(faces_t, ff, num_vertices=V)
        wa = torch.from_numpy(rng.normal(size=tuple(avg.shape)).astype(np.float32))
        (avg * wa).sum().backward()
        g[f"{name}_ff"] = ff.detach().numpy()
        g[f"{name}_average"] = avg.detach().numpy()
        g[f"{name}_average_w"] = wa.numpy()
        g[f"{name}_average_grad"] = ff.grad.numpy()
        if S == 3:
            g[f"{name}_normals"] = mm.compute_vertex_normals(faces_t, ff.detach(), num_vertices=V).numpy()
    g["cases"] = np.array(list(cases()))
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mesh_ops.npz")
    np.savez_compressed(path, **g)
    print(f"wrote {path}")


if __name__ == "__main__":
    main()
