"""Regenerate tests/golden/voxelize.npz from the reference's own trianglemeshes_to_voxelgrids and
pointclouds_to_voxelgrids, run on the CPU through oracle/ref_import.py (needs the reference sources).

Every scene stores its inputs and the reference's sparse indices, sorted and unique (4, nnz), in the
smallest int dtype that holds them, with the grid's dtype.  The maker checks that the reference's
dense grid is those indices densified, and records whether its sparse tensor is marked coalesced
(torch marks one with fewer than two entries).  Scenes
stay at resolution <= 128: the reference takes seconds per call there.

    python tests/golden/make_voxelize_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from kaolin_b200 import synthetic  # noqa: E402

CUBE_V = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float32)
CUBE_F = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1],
                   [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.int64)


def tie_mesh(res):
    """Degenerate faces (0, a, 0) along x whose float32 squared edge a*a steps through f32(thr): the
    consecutive float32 values of a around sqrt(thr), each face on its own exact y row."""
    thr = np.float32(((res - 1) / (res ** 2)) ** 2)
    a = np.float32(np.sqrt(np.float64(thr)))
    for _ in range(6):
        a = np.nextafter(a, np.float32(0))
    verts, faces = [], []
    found = set()
    for k in range(13):
        sq = np.float32(a * a)
        found.add("eq" if sq == thr else "lt" if sq < thr else "gt")
        y = np.float32(k / 16)
        base = len(verts)
        verts += [[0, y, 0], [a, y, 0], [0, y, 0]]
        faces.append([base, base + 1, base + 2])
        a = np.nextafter(a, np.float32(1))
    assert {"lt", "gt"} <= found, found
    verts.append([1, 1, 1])
    return np.array(verts, np.float32)[None], np.array(faces, np.int64)


def scenes():
    """name -> dict(kind, vertices, faces, res, origin, scale)."""
    s = {}
    f32 = np.float32

    def mesh(name, v, f, res, origin=None, scale=None):
        s[name] = dict(kind="mesh", vertices=v, faces=f, res=res, origin=origin, scale=scale)

    def pc(name, p, res, origin=None, scale=None):
        s[name] = dict(kind="pc", vertices=p, faces=None, res=res, origin=origin, scale=scale)

    mesh("doc", np.array([[[0, 0, 0], [1, 0, 0], [0, 0, 1]]], f32), np.array([[0, 1, 2]]), 3,
         np.zeros((1, 3), f32), np.ones(1, f32))
    for res in (2, 3, 4, 5, 8, 16, 32, 64):
        mesh(f"cube_{res}", CUBE_V[None], CUBE_F, res)
    v3, f3 = synthetic.icosphere(3)
    for res in (32, 128):
        mesh(f"ico3_{res}", v3[None].astype(f32), f3, res)
    v2, f2 = synthetic.icosphere(2)
    rng = np.random.default_rng(7)
    views = np.stack([v2 * (1 + 0.1 * rng.uniform(-1, 1, (v2.shape[0], 1))) + rng.normal(size=3) for _ in range(3)])
    mesh("views3", views.astype(f32), f2, 24)
    mesh("zoom", v2[None].astype(f32), f2, 32, np.full((1, 3), -0.8, f32), np.full(1, 1.0, f32))
    for res in (3, 64):
        v, f = tie_mesh(res)
        mesh(f"ties_{res}", v, f, res, np.zeros((1, 3), f32), np.ones(1, f32))
    half = np.array([[[0.125, 0.375, 0.625], [0.375, 0.625, 0.125], [0.625, 0.125, 0.375], [1, 1, 1], [0, 0, 0]]], f32)
    mesh("halfeven_5", half, np.array([[0, 0, 0], [1, 1, 2]]), 5, np.zeros((1, 3), f32), np.ones(1, f32))
    pc("pc_halfeven_5", half, 5, np.zeros((1, 3), f32), np.ones(1, f32))
    edge = np.array([[[-0.01, 0.5, 0.5], [1.01, 0.5, 0.5], [0.5, -0.1, 0.5], [0.5, 1.1, 0.5], [-0.07, 1.07, 0.2],
                      [0.5, 0.5, 0.5]]], f32)
    mesh("outside_8", edge, np.array([[0, 1, 5], [2, 3, 4]]), 8, np.zeros((1, 3), f32), np.ones(1, f32))
    pc("pc_outside_8", edge, 8, np.zeros((1, 3), f32), np.ones(1, f32))
    extra = np.concatenate([CUBE_V, [[2, 2, 2], [-0.5, 0.3, 0.7]]]).astype(f32)
    mesh("unreferenced_16", extra[None], CUBE_F, 16)
    degen = np.array([[0, 0, 0], [0, 0, 1], [1, 1, 1], [0.5, 0.5, 0.5], [1, 0, 0]], f32)
    mesh("degenerate_16", degen[None], np.array([[0, 0, 0], [0, 1, 1], [0, 3, 2], [4, 4, 2], [1, 1, 1]]), 16)
    mesh("no_faces_8", CUBE_V[None], np.zeros((0, 3), np.int64), 8)
    mesh("float64_16", CUBE_V[None].astype(np.float64), CUBE_F, 16)
    mesh("origin64_16", CUBE_V[None], CUBE_F, 16, np.zeros((1, 3), np.float64), np.ones(1, f32))
    mesh("int32_faces_16", CUBE_V[None], CUBE_F.astype(np.int32), 16)
    nan = CUBE_V.copy()
    nan[3, 1] = np.nan
    mesh("nan_default_16", nan[None], CUBE_F, 16)
    mesh("nan_explicit_16", nan[None], CUBE_F, 16, np.zeros((1, 3), f32), np.ones(1, f32))
    cloud = np.random.default_rng(11).normal(size=(2, 500, 3)).astype(f32)
    pc("pc_random_16", cloud, 16)
    pc("pc_random64_32", cloud.astype(np.float64), 32)
    pc("pc_origin64_16", cloud, 16, np.full((2, 3), -1.5, np.float64), np.full(2, 3.0, f32))
    cnan = cloud.copy()
    cnan[0, 5, 2] = np.nan
    pc("pc_nan_default_16", cnan, 16)
    pc("pc_nan_explicit_16", cnan, 16, np.full((2, 3), -2, f32), np.full(2, 4, f32))
    pc("pc_res1", cloud, 1)
    return s


def tensors(sc):
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a))
    return t(sc["vertices"]), t(sc["faces"]), t(sc["origin"]), t(sc["scale"])


def main():
    from oracle import ref_import
    pc_mod = ref_import.module("kaolin.ops.conversions.pointcloud")
    tm_mod = ref_import.module("kaolin.ops.conversions.trianglemesh")
    out = {}
    for name, sc in scenes().items():
        v, f, o, sc_ = tensors(sc)
        res = sc["res"]
        if sc["kind"] == "mesh":
            call = lambda sparse: tm_mod.trianglemeshes_to_voxelgrids(v, f, res, o, sc_, return_sparse=sparse)
        else:
            call = lambda sparse: pc_mod.pointclouds_to_voxelgrids(v, res, o, sc_, return_sparse=sparse)
        sp, dn = call(True), call(False)
        idx = sp._indices()
        assert torch.equal(idx, torch.unique(idx.T, dim=0).T), name
        ref_dense = torch.zeros(dn.shape, dtype=dn.dtype)
        ref_dense[tuple(idx)] = 1
        assert torch.equal(dn, ref_dense) and dn.dtype == sp.dtype, name
        rows = idx.numpy()
        small = np.int8 if rows.size == 0 or rows.max() < 127 else np.int16
        out[f"{name}/rows"] = rows.astype(small)
        out[f"{name}/dtype"] = np.array(str(dn.dtype).replace("torch.", ""))
        out[f"{name}/shape"] = np.array(dn.shape, np.int64)
        for k in ("vertices", "faces", "origin", "scale"):
            if sc[k] is not None:
                out[f"{name}/{k}"] = sc[k]
        out[f"{name}/res"] = np.array(res)
        out[f"{name}/coalesced"] = np.array(sp.is_coalesced())
        out[f"{name}/kind"] = np.array(sc["kind"])
        print(f"{name}: {rows.shape[1]} voxels, {dn.dtype}")
    np.savez_compressed(os.path.join(HERE, "voxelize.npz"), **out)


if __name__ == "__main__":
    main()
