"""kaolin.metrics.trianglemesh.uniform_laplacian_smoothing on sm_90a kernels, without the V x V matrix
the reference builds (trianglemesh.py:318-350)."""
import torch

from ..ops.mesh import _Topology, _apply, _check

__all__ = ["uniform_laplacian_smoothing"]


def uniform_laplacian_smoothing(vertices, faces):
    r"""Each vertex moved to the mean of its neighbours: ``(L + I) @ vertices`` for the uniform
    Laplacian L of ``faces``; vertices (B, V, 3) float32 -> (B, V, 3), with autograd to vertices.
    A vertex without neighbours goes to 0, as in the reference."""
    func = "uniform_laplacian_smoothing"
    _check(func, [("vertices", vertices, torch.float32), ("faces", faces, torch.int64)])
    topo = _Topology(func, vertices.shape[1], faces)
    return _apply(func, topo, vertices, True)
