"""Loop subdivision without a GPU: the torch restatement (oracle/subdivision.py) against the reference's
own outputs (tests/golden/subdivision.npz), the reference's signature, the C ABI's host-side argument
checks, and no CPU fallback."""
import ctypes
import inspect
import os

import numpy as np
import pytest
import torch

from kaolin_b200 import _lib
from kaolin_b200.ops import mesh
from oracle import ref_import
from oracle import subdivision as O

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "subdivision.npz"))
CASES = [str(c) for c in G["cases"]]


def rel(a, ref, scale):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(ref))
    ok = ~np.isnan(ref)
    return float(np.abs(a[ok] - ref[ok]).max(initial=0)) / max(float(scale), 1e-30)


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_the_goldens(case):
    verts = torch.from_numpy(G[f"{case}_vertices"]).double().requires_grad_(True)
    alpha = None
    if f"{case}_alpha" in G:
        alpha = torch.from_numpy(G[f"{case}_alpha"]).double().requires_grad_(True)
    out, faces = O.subdivide(verts, G[f"{case}_faces"], int(G[f"{case}_iterations"]), alpha)
    assert np.array_equal(faces.numpy(), G[f"{case}_out_faces"])
    scale = np.nanmax(np.abs(G[f"{case}_vertices"]), initial=0.0)
    assert rel(out.detach(), G[f"{case}_out"], scale) <= 1e-6
    w = torch.from_numpy(G[f"{case}_w"]).double()
    (out * w).sum().backward()
    gscale = np.nanmax(np.abs(G[f"{case}_grad_vertices"]), initial=0.0)
    assert rel(verts.grad, G[f"{case}_grad_vertices"], gscale) <= 1e-6
    if alpha is not None:
        # the scale of the terms (g . s) / n and g . x, which nearly cancel on a smooth surface
        ascale = np.nanmax(np.abs(G[f"{case}_w"]), initial=0.0) * np.nanmax(np.abs(G[f"{case}_vertices"]), initial=0.0)
        assert rel(alpha.grad, G[f"{case}_grad_alpha"], ascale) <= 1e-6


def test_oracle_reproduces_the_reference_tests_expected_tensors():
    v = torch.from_numpy(G["ref_vertices"])
    for alpha, key in ((None, "ref_expected_default"), (torch.zeros(1, 12), "ref_expected_zero_alpha")):
        out, faces = O.subdivide(v, G["ref_faces"], 1, alpha)
        assert torch.equal(faces, torch.from_numpy(G["ref_expected_faces"]))
        assert float((out - torch.from_numpy(G[key])).abs().max()) <= 1e-4


def test_oracle_rejects_out_of_range_indices():
    for bad in ([[0, 1, 3]], [[0, -1, 2]]):
        with pytest.raises(IndexError):
            O.level(3, np.array(bad))


@pytest.mark.skipif(not ref_import.available(), reason="needs the reference's sources")
def test_signature_matches_the_reference():
    theirs = ref_import.module("kaolin.ops.mesh.trianglemesh").subdivide_trianglemesh
    a, b = (inspect.signature(f).parameters for f in (mesh.subdivide_trianglemesh, theirs))
    assert [(p.name, p.default) for p in a.values()] == [(p.name, p.default) for p in b.values()]


def test_abi_rejects_bad_arguments_on_the_host():
    lib = _lib.lib()
    buf = (ctypes.c_int64 * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert lib.dibr_b200_loop_subdivision_workspace_bytes(-1, 1) == 0
    assert lib.dibr_b200_loop_subdivision_workspace_bytes(4, -1) == 0
    assert lib.dibr_b200_loop_subdivision_workspace_bytes(4, 1 << 29) == 0        # 2*F*3 does not fit 32 bits
    nbytes = lib.dibr_b200_loop_subdivision_workspace_bytes(4, 2)
    assert nbytes > 0

    def build(V=4, F=2, faces=p, ws=p, wsb=nbytes, edges=p, status=p):
        return lib.dibr_b200_loop_subdivision_build(V, F, faces, p, p, p, p, p, p, p, edges, p, status, ws, wsb, None)

    assert build(V=-1) == _lib.EINVAL
    assert build(F=-1) == _lib.EINVAL
    assert build(F=1 << 29) == _lib.ESIZE
    assert build(V=2 ** 31 - 1) == _lib.ESIZE
    assert build(faces=None) == _lib.EINVAL
    assert build(edges=None) == _lib.EINVAL
    assert build(status=None) == _lib.EINVAL
    assert build(ws=None) == _lib.EINVAL
    assert build(wsb=nbytes - 1) == _lib.EWORKSPACE

    def forward(B=1, V=4, E=5, x=p, alpha=None, alpha_out=None, edges=p):
        return lib.dibr_b200_loop_subdivision_forward(B, V, E, p, p, edges, p, x, alpha, p, alpha_out, None)

    assert forward(B=-1) == _lib.EINVAL
    assert forward(E=-1) == _lib.EINVAL
    assert forward(V=2 ** 31 - 3, E=5) == _lib.EINVAL                                 # V + E overflows
    assert forward(x=None) == _lib.EINVAL
    assert forward(edges=None) == _lib.EINVAL
    assert forward(alpha_out=p) == _lib.EINVAL                                          # no alpha to carry
    assert forward(B=0, x=None) == 0                                                    # nothing to do

    def backward(B=1, V=4, E=5, x=p, alpha=None, gao=None, gx=p, ga=None, gy=p):
        return lib.dibr_b200_loop_subdivision_backward(B, V, E, p, p, p, p, p, p, p, x, alpha, gy, gao, gx, ga, None)

    assert backward(B=-1) == _lib.EINVAL
    assert backward(gy=None) == _lib.EINVAL
    assert backward(gao=p) == _lib.EINVAL                                               # needs alpha
    assert backward(ga=p) == _lib.EINVAL                                                # needs alpha
    assert backward(alpha=p, ga=p, x=None) == _lib.EINVAL                               # needs the vertices
    assert backward(gx=None, gy=None) == 0                                              # nothing requested


def test_cpu_tensors_and_other_dtypes_raise():
    faces = torch.tensor([[0, 1, 2]])
    v = torch.rand(1, 3, 3)
    for call in (lambda: mesh.subdivide_trianglemesh(v, faces, 1),
                 lambda: mesh.subdivide_trianglemesh(v.double(), faces, 1),
                 lambda: mesh.subdivide_trianglemesh(v, faces, 1, torch.rand(1, 3)),
                 lambda: mesh.LoopSubdivision(3, faces, 1)):
        with pytest.raises(RuntimeError, match="CUDA"):
            call()
