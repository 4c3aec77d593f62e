"""Mesh Laplacian and vertex averaging without a GPU: the reference's signatures, the C ABI's host-side
argument checks, no CPU fallback, and the numpy restatement (oracle/mesh_ops.py) against the
reference's own outputs (tests/golden/mesh_ops.npz)."""
import ctypes
import inspect
import os

import numpy as np
import pytest
import torch

from kaolin_b200 import _lib
from kaolin_b200.metrics import trianglemesh
from kaolin_b200.ops import mesh
from oracle import mesh_ops as M
from oracle import ref_import

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "mesh_ops.npz"))
CASES = [str(c) for c in G["cases"]]


@pytest.mark.skipif(not ref_import.available(), reason="needs the reference's sources")
def test_signatures_match_the_reference():
    for ours, theirs, names in (
            (mesh, ref_import.module("kaolin.ops.mesh.mesh"),
             ("adjacency_matrix", "uniform_laplacian", "compute_vertex_normals", "average_face_vertex_features")),
            (trianglemesh, ref_import.module("kaolin.metrics.trianglemesh"), ("uniform_laplacian_smoothing",))):
        for name in names:
            a, b = (inspect.signature(getattr(m, name)).parameters for m in (ours, theirs))
            assert [(p.name, p.default) for p in a.values()] == [(p.name, p.default) for p in b.values()], name


def test_abi_rejects_bad_arguments_on_the_host():
    lib = _lib.lib()
    buf = (ctypes.c_int64 * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert lib.dibr_b200_mesh_topology_workspace_bytes(-1, 1, 3) == 0
    assert lib.dibr_b200_mesh_topology_workspace_bytes(4, -1, 3) == 0
    assert lib.dibr_b200_mesh_topology_workspace_bytes(4, 1, 2) == 0
    assert lib.dibr_b200_mesh_topology_workspace_bytes(4, 1 << 29, 3) == 0       # 2*F*S does not fit 32 bits
    nbytes = lib.dibr_b200_mesh_topology_workspace_bytes(4, 2, 3)
    assert nbytes > 0

    def build(V=4, F=2, S=3, faces=p, ws=p, wsb=nbytes, out=p):
        return lib.dibr_b200_mesh_topology_build(V, F, S, faces, out, p, p, p, p, p, p, ws, wsb, None)

    assert build(V=-1) == _lib.EINVAL
    assert build(F=-1) == _lib.EINVAL
    assert build(S=2) == _lib.EINVAL
    assert build(F=1 << 29) == _lib.ESIZE
    assert build(V=2 ** 31 - 1) == _lib.ESIZE
    assert build(faces=None) == _lib.EINVAL
    assert build(out=None) == _lib.EINVAL
    assert build(ws=None) == _lib.EINVAL
    assert build(wsb=nbytes - 1) == _lib.EWORKSPACE
    apply = lambda B=1, V=4, C=3, x=p: lib.dibr_b200_laplacian_apply(B, V, C, p, p, p, x, 0, 0, p, None)
    assert apply(B=-1) == _lib.EINVAL
    assert apply(C=-1) == _lib.EINVAL
    assert apply(x=None) == _lib.EINVAL
    assert apply(B=0, x=None) == 0                                                 # nothing to do
    assert lib.dibr_b200_vertex_average_forward(1, 4, 2, 3, 3, p, None, p, p, None) == _lib.EINVAL
    assert lib.dibr_b200_vertex_average_forward(1, 4, 1 << 29, 3, 3, p, p, p, p, None) == _lib.ESIZE
    assert lib.dibr_b200_vertex_average_backward(1, 4, 2, 3, -3, p, p, p, p, None) == _lib.EINVAL
    assert lib.dibr_b200_vertex_average_backward(1, 4, 2, 3, 3, None, p, p, p, None) == _lib.EINVAL
    assert lib.dibr_b200_mesh_dense(-1, 1, p, p, p, p, None) == _lib.EINVAL
    assert lib.dibr_b200_mesh_dense(4, 1, p, p, None, p, None) == _lib.EINVAL
    assert lib.dibr_b200_adjacency_coo(4, -1, p, p, p, None) == _lib.EINVAL
    assert lib.dibr_b200_adjacency_coo(4, 6, p, p, None, None) == _lib.EINVAL


def test_cpu_tensors_and_other_dtypes_raise():
    faces = torch.tensor([[0, 1, 2]])
    v = torch.rand(1, 3, 3)
    for call in (lambda: mesh.uniform_laplacian(3, faces), lambda: mesh.adjacency_matrix(3, faces),
                 lambda: mesh.UniformLaplacian(3, faces),
                 lambda: mesh.average_face_vertex_features(faces, torch.rand(1, 1, 3, 3)),
                 lambda: trianglemesh.uniform_laplacian_smoothing(v, faces)):
        with pytest.raises(RuntimeError, match="CUDA"):
            call()
    with pytest.raises(RuntimeError, match="CUDA"):
        trianglemesh.uniform_laplacian_smoothing(v.double(), faces)


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_the_goldens(case):
    t = M.topology(int(G[f"{case}_V"]), G[f"{case}_faces"])
    assert np.array_equal(M.dense_laplacian(t), G[f"{case}_laplacian"])
    assert np.array_equal(M.dense_adjacency(t), G[f"{case}_adjacency_dense"])
    assert np.array_equal(np.stack([t["rows"], t["adj"]]), G[f"{case}_adjacency_indices"])
    assert np.array_equal(M.average(t, G[f"{case}_ff"]), G[f"{case}_average"])
    F, S = G[f"{case}_faces"].shape
    assert np.array_equal(M.average_backward(t, G[f"{case}_average_w"], F, S), G[f"{case}_average_grad"])
    v, w = G[f"{case}_smooth_vertices"], G[f"{case}_smooth_w"]
    assert np.abs(M.apply(t, v, smooth=True) - G[f"{case}_smooth"]).max() <= 1e-6 * np.abs(v).max()
    g = M.apply(t, w, transpose=True, smooth=True)
    assert np.abs(g - G[f"{case}_smooth_grad"]).max() <= 1e-6 * np.abs(w).max()


def test_oracle_rejects_out_of_range_indices():
    for bad in ([[0, 1, 3]], [[0, -1, 2]]):
        with pytest.raises(IndexError):
            M.topology(3, np.array(bad))
