"""Writes tests/golden/marching_tets.npz from the reference's own marching_tetrahedra and
subdivide_tetmesh, run on the CPU (imported in place through oracle/ref_import).

Marching tetrahedra, per case <c>: V, tets, vertices (B, V, 3), sdf (B, V); the outputs of every view
concatenated (out_vertices, out_faces, tet_idx) with the per-view counts nv and nf; a weight w
(sum nv, 3); and the gradients of sum(out_vertices * w) with respect to the vertices and the sdf.
Cases: the reference test's cube of five tets with its four SDFs; one tet under all 16 sign patterns
(view c: corner k inside iff bit k of c) in four corner orders; a random tet mesh with permuted
corners, degenerate and duplicate tets and unreferenced vertices (B = 2); and that mesh with SDFs
holding exact zeros, NaN, +-inf and +-1e-38.

subdivide_tetmesh, per case <c>: vertices, tets, features (optional), the outputs, weights w and wf,
and the gradients of sum(out * w) + sum(out_features * wf).  Cases: the docstring example, and random
meshes with no features and with D = 1 and 4.

    python tests/golden/make_marching_tets_golden.py
"""
import ast
import os
import sys

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, ROOT)

from oracle import ref_import  # noqa: E402

REF_TEST = os.path.join(ref_import.REF, "tests", "python", "kaolin", "ops", "conversions", "test_tetmesh.py")
ORDERS = ["0123", "2031", "3210", "1302"]


def reference_fixtures():
    """The first tensor literal of each fixture of TestMarchingTetrahedra, by fixture name."""
    tree = ast.parse(open(REF_TEST).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "TestMarchingTetrahedra")
    out = {}
    for fn in cls.body:
        if isinstance(fn, ast.FunctionDef):
            for node in ast.walk(fn):
                if (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "tensor"
                        and node.args):
                    out[fn.name] = ast.literal_eval(node.args[0])
                    break
    return out


def random_tets(rng, V, T):
    """Random tets over V vertices: permuted corners, degenerate and duplicate tets, 3 unused vertices."""
    used = rng.permutation(V)[: V - 3]
    tets = np.stack([rng.choice(used, 4, replace=False) for _ in range(T)])
    tets[1, 2] = tets[1, 0]                     # one repeated vertex
    tets[2, :] = tets[2, 0]                     # all four the same: a self-loop only
    tets[3, 1], tets[3, 3] = tets[3, 0], tets[3, 2]   # two repeated vertices
    tets[4] = tets[5]                           # duplicate
    tets[6] = tets[7][[2, 0, 3, 1]]             # the same tet, corners permuted
    return tets.astype(np.int64)


def mt_cases(fx):
    rng = np.random.default_rng(11)
    out = {}
    cube_v = np.array(fx["vertices"], np.float32)
    out["cube"] = (np.broadcast_to(cube_v, (4,) + cube_v.shape).copy(), np.array(fx["tets"], np.int64),
                   np.array(fx["sdf"], np.float32))
    tet_v = rng.normal(size=(4, 3)).astype(np.float32)
    for order in ORDERS:
        corners = np.array([int(ch) for ch in order])
        sdf = np.empty((16, 4), np.float32)
        for c in range(16):
            for k in range(4):
                mag = rng.uniform(0.1, 2.0)
                sdf[c, corners[k]] = mag if (c >> k) & 1 else -mag
        out[f"single_{order}"] = (np.broadcast_to(tet_v, (16, 4, 3)).copy(), corners[None], sdf)
    V, T = 40, 90
    tets = random_tets(rng, V, T)
    verts = rng.normal(size=(2, V, 3)).astype(np.float32)
    out["random"] = (verts, tets, rng.normal(size=(2, V)).astype(np.float32))
    special = rng.normal(size=(2, V)).astype(np.float32)
    vals = [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-38, -1e-38]
    for b in range(2):
        pick = rng.choice(V, 14, replace=False)
        special[b, pick] = np.array(vals * 2, np.float32)
    out["special"] = (verts, tets, special)
    return out


def sub_cases():
    rng = np.random.default_rng(12)
    doc_v = np.array([[[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]]], np.float32)
    doc_f = np.array([[[-1.], [-1.], [0.5], [0.5]]], np.float32)
    out = {"sub_doc": (doc_v, np.array([[0, 1, 2, 3]], np.int64), doc_f)}
    tets = random_tets(rng, 30, 50)
    for D in (None, 1, 4):
        feats = None if D is None else rng.normal(size=(2, 30, D)).astype(np.float32)
        out[f"sub_random_{D or 0}"] = (rng.normal(size=(2, 30, 3)).astype(np.float32), tets, feats)
    return out


def main():
    conv = ref_import.module("kaolin.ops.conversions.tetmesh")
    mesh = ref_import.module("kaolin.ops.mesh.tetmesh")
    rng = np.random.default_rng(13)
    g = {}
    mcases = mt_cases(reference_fixtures())
    for name, (verts, tets, sdf) in mcases.items():
        v = torch.from_numpy(verts).requires_grad_(True)
        s = torch.from_numpy(sdf).requires_grad_(True)
        ov, of, ot = conv.marching_tetrahedra(v, torch.from_numpy(tets), s, True)
        flat = torch.cat(ov)
        w = rng.normal(size=tuple(flat.shape)).astype(np.float32)
        if flat.numel():
            (flat * torch.from_numpy(w)).sum().backward()
        g[f"{name}_V"] = np.int64(verts.shape[1])
        g[f"{name}_tets"] = tets
        g[f"{name}_vertices"] = verts
        g[f"{name}_sdf"] = sdf
        g[f"{name}_out_vertices"] = flat.detach().numpy()
        g[f"{name}_nv"] = np.array([len(x) for x in ov], np.int64)
        g[f"{name}_out_faces"] = torch.cat(of).numpy().astype(np.int32)
        g[f"{name}_nf"] = np.array([len(x) for x in of], np.int64)
        g[f"{name}_tet_idx"] = torch.cat(ot).numpy().astype(np.int32)
        g[f"{name}_w"] = w
        g[f"{name}_grad_vertices"] = np.zeros_like(verts) if v.grad is None else v.grad.numpy()
        g[f"{name}_grad_sdf"] = np.zeros_like(sdf) if s.grad is None else s.grad.numpy()
    scases = sub_cases()
    for name, (verts, tets, feats) in scases.items():
        v = torch.from_numpy(verts).requires_grad_(True)
        f = None if feats is None else torch.from_numpy(feats).requires_grad_(True)
        out = mesh.subdivide_tetmesh(v, torch.from_numpy(tets), f)
        w = rng.normal(size=tuple(out[0].shape)).astype(np.float32)
        loss = (out[0] * torch.from_numpy(w)).sum()
        g[f"{name}_vertices"] = verts
        g[f"{name}_tets"] = tets
        g[f"{name}_out_vertices"] = out[0].detach().numpy()
        g[f"{name}_out_tets"] = out[1].numpy().astype(np.int32)
        g[f"{name}_w"] = w
        if f is not None:
            wf = rng.normal(size=tuple(out[2].shape)).astype(np.float32)
            loss = loss + (out[2] * torch.from_numpy(wf)).sum()
            g[f"{name}_features"] = feats
            g[f"{name}_out_features"] = out[2].detach().numpy()
            g[f"{name}_wf"] = wf
        loss.backward()
        g[f"{name}_grad_vertices"] = v.grad.numpy()
        if f is not None:
            g[f"{name}_grad_features"] = f.grad.numpy()
    g["mt_cases"] = np.array(list(mcases))
    g["sub_cases"] = np.array(list(scases))
    g["single_orders"] = np.array(ORDERS)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "marching_tets.npz")
    np.savez_compressed(path, **g)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
