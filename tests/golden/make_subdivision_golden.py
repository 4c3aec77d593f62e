"""Writes tests/golden/subdivision.npz from the reference's own subdivide_trianglemesh, run on the CPU
(imported in place through oracle/ref_import).  The reference handles one view per call, so a batched
case is per-view calls, stacked.

Per case <c>: V, faces, iterations, vertices (B, V, 3), alpha (B, V) when given, the output vertices and
faces, a weight w, and the gradients of sum(out * w) with respect to the vertices and alpha.  Also the
icosahedron and the expected tensors of the reference's TestSubdivideTrianglemesh (read from its test
file), and the total face area it expects after 5 iterations.

    python tests/golden/make_subdivision_golden.py
"""
import ast
import os
import sys

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, ROOT)

from oracle import ref_import  # noqa: E402
from kaolin_b200 import synthetic  # noqa: E402

REF_TEST = os.path.join(ref_import.REF, "tests", "python", "kaolin", "ops", "mesh", "test_trianglemesh.py")


def reference_fixtures():
    """The tensor literals of TestSubdivideTrianglemesh's fixtures, by fixture name."""
    tree = ast.parse(open(REF_TEST).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "TestSubdivideTrianglemesh")
    out = {}
    for fn in cls.body:
        if isinstance(fn, ast.FunctionDef) and isinstance(fn.body[-1], ast.Return):
            call = fn.body[-1].value
            if isinstance(call, ast.Call) and call.args:
                out[fn.name] = ast.literal_eval(call.args[0])
    return out


def random_mesh(rng, V, F):
    """Random triangles over V vertices with degenerate faces, duplicate faces and unreferenced vertices."""
    used = rng.permutation(V)[: V - 3]                 # three vertices referenced by no face
    faces = rng.choice(used, size=(F, 3))
    faces[1, 1] = faces[1, 0]                          # degenerate: a repeated vertex
    faces[2, :] = faces[2, 0]                          # fully degenerate: a self-loop only
    faces[3] = faces[4]                                # duplicate face
    faces[5] = np.roll(faces[6], 1)                    # the same face, rotated
    return faces


def cases(fx):
    rng = np.random.default_rng(99)
    ico_v = np.array(fx["vertices_icosahedron"], np.float32)
    ico_f = np.array(fx["faces_icosahedron"], np.int64)
    # an open strip (boundary edges), a fin on edge (1, 2) (three faces), a face (1, 1, 5) with a
    # self-loop, and vertex 7 referenced by no face
    open_f = np.array([[0, 1, 2], [1, 3, 2], [2, 3, 4], [1, 2, 5], [3, 6, 4], [1, 1, 5]], np.int64)
    rand_f = random_mesh(rng, 64, 120)
    v3, f3 = synthetic.icosphere(3)
    f3 = np.asarray(f3, np.int64)
    # name: (vertices (B, V, 3), faces, iterations, alpha (B, V) or None)
    out = {
        "ico_default": (ico_v, ico_f, 1, None),
        "ico_zero_alpha": (ico_v, ico_f, 1, np.zeros((1, 12), np.float32)),
        "ico_alpha_2iter": (ico_v, ico_f, 2, rng.uniform(0, 1, (1, 12)).astype(np.float32)),
        "random": (rng.normal(size=(2, 64, 3)).astype(np.float32), rand_f, 2, None),
        "random_alpha": (rng.normal(size=(2, 64, 3)).astype(np.float32), rand_f, 2,
                         rng.uniform(0, 1, (2, 64)).astype(np.float32)),
        "open": (rng.normal(size=(2, 8, 3)).astype(np.float32), open_f, 2, None),
        "open_alpha": (rng.normal(size=(2, 8, 3)).astype(np.float32), open_f, 2,
                       rng.uniform(0, 1, (2, 8)).astype(np.float32)),
        "empty": (rng.normal(size=(2, 4, 3)).astype(np.float32), np.zeros((0, 3), np.int64), 1, None),
        "empty_alpha": (rng.normal(size=(2, 4, 3)).astype(np.float32), np.zeros((0, 3), np.int64), 1,
                        np.zeros((2, 4), np.float32)),
    }
    for it in (1, 2):
        out[f"ico3_{it}iter"] = (np.asarray(v3, np.float32)[None], f3, it, None)
        out[f"ico3_{it}iter_alpha"] = (np.asarray(v3, np.float32)[None], f3, it,
                                       rng.uniform(0, 1, (1, len(v3))).astype(np.float32))
    return out


def main():
    tm = ref_import.module("kaolin.ops.mesh.trianglemesh")
    fx = reference_fixtures()
    rng = np.random.default_rng(7)
    g = {
        "ref_vertices": np.array(fx["vertices_icosahedron"], np.float32),
        "ref_faces": np.array(fx["faces_icosahedron"], np.int64),
        "ref_expected_default": np.array(fx["expected_vertices_default_alpha"], np.float32),
        "ref_expected_zero_alpha": np.array(fx["expected_vertices_zero_alpha"], np.float32),
        "ref_expected_faces": np.array(fx["expected_faces_icosahedron_1_iter"], np.int64),
    }
    v5, f5 = tm.subdivide_trianglemesh(torch.from_numpy(g["ref_vertices"]), torch.from_numpy(g["ref_faces"]), 5)
    g["ref_5iter_area"] = np.float32(tm.face_areas(v5, f5).sum())
    g["ref_5iter_faces"] = np.int64(f5.shape[0])
    all_cases = cases(fx)
    for name, (verts, faces, iterations, alpha) in all_cases.items():
        B, V = verts.shape[:2]
        outs, gvs, gas, w = [], [], [], None
        for b in range(B):                       # the reference takes one view per call
            v = torch.from_numpy(verts[b:b + 1].copy()).requires_grad_(True)
            a = None if alpha is None else torch.from_numpy(alpha[b:b + 1].copy()).requires_grad_(True)
            out, out_faces = tm.subdivide_trianglemesh(v, torch.from_numpy(faces), iterations, a)
            if w is None:
                w = rng.normal(size=(B,) + tuple(out.shape[1:])).astype(np.float32)
            (out * torch.from_numpy(w[b:b + 1])).sum().backward()
            outs.append(out.detach().numpy())
            gvs.append(v.grad.numpy())
            if a is not None:
                gas.append(a.grad.numpy())
        g[f"{name}_V"] = np.int64(V)
        g[f"{name}_faces"] = faces
        g[f"{name}_iterations"] = np.int64(iterations)
        g[f"{name}_vertices"] = verts
        g[f"{name}_out"] = np.concatenate(outs)
        g[f"{name}_out_faces"] = out_faces.numpy().astype(np.int32)
        g[f"{name}_w"] = w
        g[f"{name}_grad_vertices"] = np.concatenate(gvs)
        if alpha is not None:
            g[f"{name}_alpha"] = alpha
            g[f"{name}_grad_alpha"] = np.concatenate(gas)
    g["cases"] = np.array(list(all_cases))
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "subdivision.npz")
    np.savez_compressed(path, **g)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
