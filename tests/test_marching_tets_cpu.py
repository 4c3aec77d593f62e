"""Marching tetrahedra and subdivide_tetmesh without a GPU: the torch restatement
(oracle/marching_tets.py) against the reference's own outputs (tests/golden/marching_tets.npz), the
reference's signatures, the library's case table, the C ABI's host-side argument checks, and no CPU
fallback."""
import ctypes
import inspect
import os

import numpy as np
import pytest
import torch

from kaolin_b200 import _lib
from kaolin_b200.ops import conversions, mesh
from kaolin_b200.ops.conversions import tetmesh
from oracle import marching_tets as O
from oracle import ref_import

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "marching_tets.npz"))
MT_CASES = [str(c) for c in G["mt_cases"]]
SUB_CASES = [str(c) for c in G["sub_cases"]]


def golden_table():
    return O.case_table(G["single_0123_out_faces"], G["single_0123_nf"])


def rel(a, ref, scale):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(ref)), "NaN positions differ"
    ok = ~np.isnan(ref)
    assert np.array_equal(a[ok & np.isinf(ref)], ref[ok & np.isinf(ref)])
    ok &= ~np.isinf(ref)
    return float(np.abs(a[ok] - ref[ok]).max(initial=0)) / max(float(scale), 1e-30)


def finite_max(a):
    a = np.abs(np.asarray(a, np.float64))
    return float(a[np.isfinite(a)].max(initial=0.0))


@pytest.mark.parametrize("case", MT_CASES)
def test_oracle_reproduces_the_marching_goldens(case):
    table = golden_table()
    for dtype in (torch.float32, torch.float64):
        v = torch.from_numpy(G[f"{case}_vertices"]).to(dtype).requires_grad_(True)
        s = torch.from_numpy(G[f"{case}_sdf"]).to(dtype).requires_grad_(True)
        out = O.marching(v, G[f"{case}_tets"], s, table)
        assert [len(o[0]) for o in out] == list(G[f"{case}_nv"])
        assert torch.equal(torch.cat([o[1] for o in out]), torch.from_numpy(G[f"{case}_out_faces"].astype(np.int64)))
        assert torch.equal(torch.cat([o[2] for o in out]), torch.from_numpy(G[f"{case}_tet_idx"].astype(np.int64)))
        flat = torch.cat([o[0] for o in out])
        if dtype == torch.float32:       # the same element-wise steps in the same precision: bit-equal
            assert np.array_equal(flat.detach().numpy(), G[f"{case}_out_vertices"], equal_nan=True)
        elif case != "special":          # +-1e-38 and infinities round differently in fp64
            assert rel(flat.detach(), G[f"{case}_out_vertices"], finite_max(G[f"{case}_vertices"])) <= 1e-6
        if flat.numel() and (dtype == torch.float32 or case != "special"):
            (flat * torch.from_numpy(G[f"{case}_w"]).to(dtype)).sum().backward()
            for got, key in ((v.grad, "grad_vertices"), (s.grad, "grad_sdf")):
                assert rel(got, G[f"{case}_{key}"], finite_max(G[f"{case}_{key}"])) <= 1e-6


@pytest.mark.parametrize("case", MT_CASES)
def test_device_restatement_reproduces_the_marching_goldens(case):
    """The torch-only restatement of the reference's structure (the benchmark's baseline) gives the
    reference's outputs, the fp32 vertices bit for bit."""
    out = O.marching_on_device(torch.from_numpy(G[f"{case}_vertices"]), G[f"{case}_tets"],
                               torch.from_numpy(G[f"{case}_sdf"]), golden_table())
    assert np.array_equal(torch.cat([o[0] for o in out]).numpy(), G[f"{case}_out_vertices"], equal_nan=True)
    assert torch.equal(torch.cat([o[1] for o in out]), torch.from_numpy(G[f"{case}_out_faces"].astype(np.int64)))
    assert torch.equal(torch.cat([o[2] for o in out]), torch.from_numpy(G[f"{case}_tet_idx"].astype(np.int64)))


@pytest.mark.parametrize("case", SUB_CASES)
def test_oracle_reproduces_the_subdivision_goldens(case):
    v = torch.from_numpy(G[f"{case}_vertices"]).double().requires_grad_(True)
    f = torch.from_numpy(G[f"{case}_features"]).double().requires_grad_(True) if f"{case}_features" in G else None
    y, tets, yf = O.subdivide(v, G[f"{case}_tets"], f)
    assert np.array_equal(tets.numpy(), G[f"{case}_out_tets"])
    assert rel(y.detach(), G[f"{case}_out_vertices"], finite_max(G[f"{case}_vertices"])) <= 1e-7
    loss = (y * torch.from_numpy(G[f"{case}_w"]).double()).sum()
    if f is not None:
        assert rel(yf.detach(), G[f"{case}_out_features"], finite_max(G[f"{case}_features"])) <= 1e-7
        loss = loss + (yf * torch.from_numpy(G[f"{case}_wf"]).double()).sum()
    loss.backward()
    assert rel(v.grad, G[f"{case}_grad_vertices"], finite_max(G[f"{case}_grad_vertices"])) <= 1e-6
    if f is not None:
        assert rel(f.grad, G[f"{case}_grad_features"], finite_max(G[f"{case}_grad_features"])) <= 1e-6


def test_every_corner_order_of_one_tet_follows_the_table():
    """The golden's single tet in every corner order: the oracle (with the table read off order 0123)
    gives the reference's faces, so the table is one of corners, not of vertex numbers."""
    for order in (str(o) for o in G["single_orders"]):
        case = f"single_{order}"
        out = O.marching(torch.from_numpy(G[f"{case}_vertices"]), G[f"{case}_tets"],
                         torch.from_numpy(G[f"{case}_sdf"]), golden_table())
        assert torch.equal(torch.cat([o[1] for o in out]), torch.from_numpy(G[f"{case}_out_faces"].astype(np.int64)))


def test_library_case_table_is_the_references():
    pairs = tetmesh.case_table().numpy()              # (16, 2, 3, 2) corners, -1 where unused
    table = golden_table()
    for c in range(16):
        for k in range(2):
            for u in range(3):
                i, j = pairs[c, k, u]
                if table[c, k, u] < 0:
                    assert i == j == -1
                else:
                    assert [i, j] == list(O.PAIRS[table[c, k, u]])


def test_every_edge_a_case_uses_has_a_sign_change():
    pairs = tetmesh.case_table().numpy()
    for c in range(16):
        occ = [(c >> k) & 1 for k in range(4)]
        inside = sum(occ)
        used = pairs[c][pairs[c, :, :, 0] >= 0]
        assert len(used) == 3 * {0: 0, 1: 1, 2: 2, 3: 1, 4: 0}[inside]
        for i, j in used:
            assert i < j and occ[i] != occ[j], (c, i, j)


def test_oracle_rejects_out_of_range_indices():
    for bad in ([[0, 1, 2, 4]], [[0, -1, 2, 3]]):
        with pytest.raises(IndexError):
            O.topology(4, np.array(bad))


@pytest.mark.skipif(not ref_import.available(), reason="needs the reference's sources")
def test_signatures_match_the_reference():
    pairs = ((conversions.marching_tetrahedra, "kaolin.ops.conversions.tetmesh", "marching_tetrahedra"),
             (mesh.subdivide_tetmesh, "kaolin.ops.mesh.tetmesh", "subdivide_tetmesh"))
    for ours, mod, name in pairs:
        theirs = getattr(ref_import.module(mod), name)
        a, b = (inspect.signature(f).parameters for f in (ours, theirs))
        assert [(p.name, p.default) for p in a.values()] == [(p.name, p.default) for p in b.values()]


def test_abi_rejects_bad_arguments_on_the_host():
    lib = _lib.lib()
    buf = (ctypes.c_int64 * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert lib.dibr_b200_tet_topology_workspace_bytes(-1, 1) == 0
    assert lib.dibr_b200_tet_topology_workspace_bytes(4, -1) == 0
    assert lib.dibr_b200_tet_topology_workspace_bytes(4, 1 << 28) == 0          # 12 T does not fit 32 bits
    nbytes = lib.dibr_b200_tet_topology_workspace_bytes(4, 2)
    assert nbytes > 0

    def build(V=4, T=2, tets=p, ws=p, wsb=nbytes, edges=p, status=p):
        return lib.dibr_b200_tet_topology_build(V, T, tets, p, p, edges, p, p, status, ws, wsb, None)

    assert build(V=-1) == _lib.EINVAL
    assert build(T=-1) == _lib.EINVAL
    assert build(T=1 << 28) == _lib.ESIZE
    assert build(V=2 ** 31 - 1) == _lib.ESIZE
    assert build(tets=None) == _lib.EINVAL
    assert build(edges=None) == _lib.EINVAL
    assert build(status=None) == _lib.EINVAL
    assert build(ws=None) == _lib.EINVAL
    assert build(wsb=nbytes - 1) == _lib.EWORKSPACE

    assert lib.dibr_b200_marching_tets_workspace_bytes(-1, 5, 2) == 0
    assert lib.dibr_b200_marching_tets_workspace_bytes(8, 1 << 28, 1 << 26) == 0   # B (E + 2T) overflows
    mbytes = lib.dibr_b200_marching_tets_workspace_bytes(2, 5, 2)
    assert mbytes > 0

    def count(B=2, V=4, E=5, T=2, edges=p, tets=p, sdf=p, scan=p, counts=p, ws=p, wsb=mbytes):
        return lib.dibr_b200_marching_tets_count(B, V, E, T, edges, tets, sdf, scan, counts, ws, wsb, None)

    assert count(B=-1) == _lib.EINVAL
    assert count(E=1 << 30) == _lib.ESIZE
    assert count(edges=None) == _lib.EINVAL
    assert count(tets=None) == _lib.EINVAL
    assert count(sdf=None) == _lib.EINVAL
    assert count(scan=None) == _lib.EINVAL
    assert count(counts=None) == _lib.EINVAL
    assert count(wsb=mbytes - 1) == _lib.EWORKSPACE

    def emit(B=2, V=4, E=5, T=2, edges=p, x=p, sdf=p, scan=p, vid=p, ov=p, of=p):
        return lib.dibr_b200_marching_tets_emit(B, V, E, T, edges, p, p, x, sdf, scan, vid, ov, of, None, None)

    assert emit(B=-1) == _lib.EINVAL
    assert emit(x=None) == _lib.EINVAL
    assert emit(scan=None) == _lib.EINVAL
    assert emit(vid=None) == _lib.EINVAL
    assert emit(ov=None) == _lib.EINVAL
    assert emit(B=0, x=None, scan=None) == 0                                         # nothing to do

    def backward(B=2, V=4, E=5, x=p, sdf=p, vid=p, g=p, gx=p, gs=p):
        return lib.dibr_b200_marching_tets_backward(B, V, E, p, p, p, x, sdf, vid, g, gx, gs, None)

    assert backward(B=-1) == _lib.EINVAL
    assert backward(x=None) == _lib.EINVAL
    assert backward(vid=None) == _lib.EINVAL
    assert backward(g=None) == _lib.EINVAL
    assert backward(gx=None, gs=None, x=None) == 0                                  # nothing requested

    def sub_fwd(B=1, V=4, E=6, T=1, D=0, edges=p, x=p, f=None, y=p, yf=None, out_tets=p, tets=p):
        return lib.dibr_b200_tet_subdivide_forward(B, V, E, T, D, edges, tets, p, x, f, y, yf, out_tets, None)

    assert sub_fwd(B=-1) == _lib.EINVAL
    assert sub_fwd(V=2 ** 31 - 3, E=5) == _lib.ESIZE                                   # V + E overflows
    assert sub_fwd(T=1 << 28) == _lib.ESIZE                                             # 12 T overflows
    assert sub_fwd(x=None) == _lib.EINVAL
    assert sub_fwd(edges=None) == _lib.EINVAL
    assert sub_fwd(D=2) == _lib.EINVAL                                                  # features missing
    assert sub_fwd(tets=None) == _lib.EINVAL

    def sub_bwd(B=1, V=4, E=6, D=0, gy=p, gyf=None, gx=p, gf=None):
        return lib.dibr_b200_tet_subdivide_backward(B, V, E, D, p, p, p, gy, gyf, gx, gf, None)

    assert sub_bwd(B=-1) == _lib.EINVAL
    assert sub_bwd(V=2 ** 31 - 3, E=5) == _lib.ESIZE                                   # V + E overflows
    assert sub_bwd(gy=None) == _lib.EINVAL
    assert sub_bwd(D=2, gf=p) == _lib.EINVAL                                            # grad_out features missing
    assert sub_bwd(gx=None) == 0                                                       # nothing requested
    assert lib.dibr_b200_marching_tets_case_table(None) == _lib.EINVAL


def test_cpu_tensors_and_other_dtypes_raise():
    tets = torch.tensor([[0, 1, 2, 3]])
    v, s = torch.rand(1, 4, 3), torch.rand(1, 4)
    for call in (lambda: conversions.marching_tetrahedra(v, tets, s),
                 lambda: conversions.marching_tetrahedra(v.double(), tets, s),
                 lambda: conversions.MarchingTetrahedra(4, tets),
                 lambda: mesh.subdivide_tetmesh(v, tets),
                 lambda: mesh.subdivide_tetmesh(v, tets, torch.rand(1, 4, 2))):
        with pytest.raises(RuntimeError, match="CUDA"):
            call()
