"""Mesh Laplacian, adjacency and vertex averaging on sm_90a (csrc/mesh_topology.cu) against the
reference's own outputs (tests/golden/mesh_ops.npz) and the fp64 restatement (oracle/mesh_ops.py):
exact where the reference's arithmetic is reproduced (dense matrices, sparse indices, averaging),
within 1e-6 of scale for the Laplacian products; plus edge cases, determinism, no host
synchronisation, c5's 1.3 M-face mesh, and one DIB-R tutorial step with the Laplacian regulariser."""
import math
import os

import numpy as np
import pytest
import torch

from kaolin_b200 import _lib, synthetic
from kaolin_b200.metrics import trianglemesh
from kaolin_b200.metrics.render import mask_iou
from kaolin_b200.ops import mesh
from kaolin_b200.render.mesh import dibr_rasterization, prepare_vertices, texture_mapping
from oracle import mesh_ops as M

pytestmark = pytest.mark.gpu
DEV = "cuda"
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "mesh_ops.npz"))
CASES = [str(c) for c in G["cases"]]
T = lambda a, grad=False: torch.from_numpy(np.ascontiguousarray(a)).to(DEV).requires_grad_(grad)


def traced(fn):
    _lib.trace_begin()
    try:
        out = fn()
    finally:
        ran = [name for name, _ in _lib.trace_end(1024)]
    return out, ran


def rel(a, ref, scale):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    return float(np.abs(a.astype(np.float64) - ref).max()) / max(float(scale), 1e-30)


def fan(n):
    """One vertex in n triangles (0, i+1, i+2): its row has n corners and n+1 neighbours."""
    return n + 2, np.stack([np.zeros(n, np.int64), np.arange(1, n + 1), np.arange(2, n + 2)], 1)


@pytest.mark.parametrize("case", CASES)
def test_exact_against_the_reference(case):
    V, faces = int(G[f"{case}_V"]), T(G[f"{case}_faces"])
    (L, ran) = traced(lambda: mesh.uniform_laplacian(V, faces))
    assert torch.equal(L.cpu(), torch.from_numpy(G[f"{case}_laplacian"]))
    assert "dense_kernel<laplacian>" in ran and "topo_compact_kernel" in ran
    assert torch.equal(mesh.adjacency_matrix(V, faces, sparse=False).cpu(), torch.from_numpy(G[f"{case}_adjacency_dense"]))
    sp = mesh.adjacency_matrix(V, faces)
    assert (not sp.is_coalesced() or sp._nnz() < 2) and tuple(sp.shape) == (V, V)   # torch marks nnz < 2 coalesced
    assert torch.equal(sp._indices().cpu(), torch.from_numpy(G[f"{case}_adjacency_indices"]))
    assert torch.equal(sp._values().cpu(), torch.from_numpy(G[f"{case}_adjacency_values"]))
    assert torch.equal(mesh.UniformLaplacian(V, faces).to_dense().cpu(), torch.from_numpy(G[f"{case}_laplacian"]))

    ff = T(G[f"{case}_ff"], True)
    (avg, ran) = traced(lambda: mesh.average_face_vertex_features(faces, ff, num_vertices=V))
    assert "vertex_average_kernel" in ran
    assert torch.equal(avg.detach().cpu(), torch.from_numpy(G[f"{case}_average"]))
    (avg * T(G[f"{case}_average_w"])).sum().backward()
    assert torch.equal(ff.grad.cpu(), torch.from_numpy(G[f"{case}_average_grad"]))
    if f"{case}_normals" in G:
        n = mesh.compute_vertex_normals(faces, ff.detach(), num_vertices=V)
        assert torch.equal(n.cpu(), torch.from_numpy(G[f"{case}_normals"]))


@pytest.mark.parametrize("case", CASES)
def test_smoothing_and_products_within_tolerance(case):
    V, faces_np = int(G[f"{case}_V"]), G[f"{case}_faces"]
    faces = T(faces_np)
    t = M.topology(V, faces_np)
    v = T(G[f"{case}_smooth_vertices"], True)
    w = G[f"{case}_smooth_w"]
    (s, ran) = traced(lambda: trianglemesh.uniform_laplacian_smoothing(v, faces))
    assert "laplacian_apply3_kernel<smooth>" in ran
    scale = np.abs(G[f"{case}_smooth_vertices"]).max()
    assert rel(s, G[f"{case}_smooth"], scale) <= 1e-6
    assert rel(s, M.apply(t, G[f"{case}_smooth_vertices"], smooth=True), scale) <= 1e-6
    s.backward(T(w))
    assert rel(v.grad, G[f"{case}_smooth_grad"], np.abs(w).max()) <= 1e-6
    assert rel(v.grad, M.apply(t, w, transpose=True, smooth=True), np.abs(w).max()) <= 1e-6

    L = mesh.UniformLaplacian(V, faces)
    Ld = torch.from_numpy(G[f"{case}_laplacian"]).double()
    for shape in ((V, 3), (2, V, 3), (V, 5), (3, V, 1)):
        x = torch.randn(shape, dtype=torch.float32).to(DEV).requires_grad_(True)
        g = torch.randn(shape, dtype=torch.float32)
        y = L @ x
        y.backward(g.to(DEV))
        ref = torch.matmul(Ld, x.detach().cpu().double())
        assert rel(y, ref.numpy(), x.abs().max()) <= 1e-6
        assert rel(y, M.apply(t, x.detach().cpu().numpy()), x.abs().max()) <= 1e-6
        assert rel(x.grad, torch.matmul(Ld.t(), g.double()).numpy(), g.abs().max()) <= 1e-6
        assert torch.equal(L.matmul(x.detach()), y.detach())


def test_reference_tests_expected_tensors():
    faces = T(np.array([[1, 3, 2], [1, 4, 0]]))
    assert torch.equal(mesh.uniform_laplacian(5, faces).cpu(), torch.tensor(
        [[-1, 0.5, 0, 0, 0.5], [0.25, -1, 0.25, 0.25, 0.25], [0, 0.5, -1, 0.5, 0], [0, 0.5, 0.5, -1, 0],
         [0.5, 0.5, 0, 0, -1]]))
    r = mesh.uniform_laplacian(4, T(np.array([[0, 1, 2]]))).cpu()
    assert torch.equal(r[3, :3], torch.zeros(3)) and torch.equal(r[:3, 3], torch.zeros(3))
    v = T(np.array([[[0, 0, 1], [2, 1, 2], [3, 1, 2]], [[3, 1, 2], [0, 0, 3], [0, 3, 3]]], np.float32))
    out = trianglemesh.uniform_laplacian_smoothing(v, T(np.array([[0, 1, 2]])))
    assert torch.equal(out.cpu(), torch.tensor([[[2.5, 1.0, 2.0], [1.5, 0.5, 1.5], [1.0, 0.5, 1.5]],
                                                [[0.0, 1.5, 3.0], [1.5, 2.0, 2.5], [1.5, 0.5, 2.5]]]))
    fn = T(np.array([[0, 2, 1], [0, 3, 2], [0, 4, 3]]))
    nrm = torch.rand((3, 3, 3, 3), device=DEV)
    a = mesh.compute_vertex_normals(fn, nrm)                  # num_vertices from faces.max(): V = 5
    assert a.shape == (3, 5, 3)
    assert torch.equal(a[:, 1], nrm[:, 0, 2]) and torch.equal(a[:, 2], (nrm[:, 0, 1] + nrm[:, 1, 2]) / 2)


def test_topology_matches_the_oracle_csr_and_edge_cases():
    for case in CASES:
        V, faces_np = int(G[f"{case}_V"]), G[f"{case}_faces"]
        topo = mesh._Topology("test", V, T(faces_np))
        t = M.topology(V, faces_np)
        for k in ("corner_ptr", "corners", "adj_ptr", "adj", "degree"):
            assert np.array_equal(getattr(topo, k).cpu().numpy()[:len(t[k])], t[k]), (case, k)
        assert np.array_equal(topo.weight.cpu().numpy(), t["weight"]), case
    # F = 0: L = -I, smoothing gives 0, averaging 0
    e = T(np.zeros((0, 3), np.int64))
    assert torch.equal(mesh.uniform_laplacian(4, e).cpu(), -torch.eye(4))
    assert mesh.adjacency_matrix(4, e)._nnz() == 0
    v = torch.rand((2, 4, 3), device=DEV)
    assert torch.equal(trianglemesh.uniform_laplacian_smoothing(v, e), torch.zeros_like(v))
    assert torch.equal(mesh.average_face_vertex_features(e, torch.zeros((2, 0, 3, 3), device=DEV), 4),
                       torch.zeros((2, 4, 3), device=DEV))
    # a face of one repeated vertex: a self-loop, degree 1, L row -1 on the diagonal, smoothed to 0
    L = mesh.uniform_laplacian(3, T(np.array([[2, 2, 2]]))).cpu()
    assert torch.equal(L, -torch.eye(3))
    assert torch.equal(mesh.adjacency_matrix(3, T(np.array([[2, 2, 2]])), sparse=False).cpu()[2], torch.tensor([0., 0., 1.]))


@pytest.mark.parametrize("bad", [[[0, 1, 5]], [[0, -1, 2]], [[0, 1, 2], [3, 1, 1 << 40]]])
def test_out_of_range_index_raises_and_writes_nothing(bad):
    v = torch.rand((1, 4, 3), device=DEV)
    guard = torch.full((1 << 16,), 7.0, device=DEV)
    for call in (lambda: mesh.uniform_laplacian(4, T(np.array(bad))),
                 lambda: mesh.adjacency_matrix(4, T(np.array(bad))),
                 lambda: mesh.UniformLaplacian(4, T(np.array(bad))),
                 lambda: trianglemesh.uniform_laplacian_smoothing(v, T(np.array(bad))),
                 lambda: mesh.average_face_vertex_features(T(np.array(bad)), torch.rand((1, len(bad), 3, 3), device=DEV), 4)):
        with pytest.raises(IndexError):
            call()
    torch.cuda.synchronize()
    assert bool((guard == 7.0).all())


def test_fan_vertex_long_rows():
    V, faces_np = fan(10000)
    faces = T(faces_np)
    t = M.topology(V, faces_np)
    topo = mesh._Topology("test", V, faces)
    assert np.array_equal(topo.adj.cpu().numpy(), t["adj"]) and np.array_equal(topo.corners.cpu().numpy(), t["corners"])
    assert int(topo.degree[0]) == 10001
    gen = torch.Generator(device="cpu").manual_seed(0)
    x = (torch.rand((2, V, 3), generator=gen) * 2 - 1)
    L = mesh.UniformLaplacian(V, faces)
    xd = x.to(DEV).requires_grad_(True)
    y = L @ xd
    y.backward(x.to(DEV))
    deg = t["degree"].astype(np.float64)
    bound = (deg + 2)[None, :, None] * 2.0 ** -24 * float(x.abs().max())
    assert np.all(np.abs(y.detach().cpu().numpy() - M.apply(t, x.numpy())) <= bound)
    assert np.all(np.abs(xd.grad.cpu().numpy() - M.apply(t, x.numpy(), transpose=True)) <= bound)
    ff = torch.randn((1, len(faces_np), 3, 3), generator=gen)
    assert np.array_equal(mesh.average_face_vertex_features(faces, ff.to(DEV)).cpu().numpy(), M.average(t, ff.numpy()))


def test_runs_are_byte_identical():
    V, f = synthetic.icosphere(4)
    faces_np = np.concatenate([np.asarray(f), fan(300)[1]])            # a long row among short ones
    V = max(len(V), 302)
    faces = T(faces_np)
    gen = torch.Generator(device="cpu").manual_seed(1)
    x = torch.randn((4, V, 3), generator=gen).to(DEV)
    g = torch.randn((4, V, 3), generator=gen).to(DEV)
    ff = torch.randn((2, len(faces_np), 3, 7), generator=gen).to(DEV)

    def run():
        L = mesh.UniformLaplacian(V, faces)
        xs = [x.clone().requires_grad_(True), x[..., :2].contiguous().requires_grad_(True)]
        outs = []
        for xi in xs:
            y = L @ xi
            y.backward(g[..., :xi.shape[-1]])
            outs += [y.detach(), xi.grad]
        v = x.clone().requires_grad_(True)
        s = trianglemesh.uniform_laplacian_smoothing(v, faces)
        s.backward(g)
        fr = ff.clone().requires_grad_(True)
        a = mesh.average_face_vertex_features(faces, fr, V)
        a.backward(torch.ones_like(a))
        return outs + [s.detach(), v.grad, a.detach(), fr.grad, L.to_dense(),
                       mesh.adjacency_matrix(V, faces)._indices()]

    for a, b in zip(run(), run()):
        assert torch.equal(a, b)


def test_apply_makes_no_host_synchronisation():
    V, f = synthetic.icosphere(3)
    faces = T(np.asarray(f))
    L = mesh.UniformLaplacian(len(V), faces)
    x = torch.randn((2, len(V), 3), device=DEV, requires_grad=True)
    g = torch.randn((2, len(V), 3), device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        y = L @ x
        y.backward(g)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert x.grad is not None


def test_c5_mesh_in_bounded_memory():
    verts, f = synthetic.icosphere(8)
    V, faces_np = len(verts), np.asarray(f, np.int64)
    assert len(faces_np) == 1310720
    faces = T(faces_np)
    B = 32
    gen = torch.Generator(device="cpu").manual_seed(2)
    x = torch.randn((B, V, 3), generator=gen).to(DEV).requires_grad_(True)
    g = torch.randn((B, V, 3), generator=gen).to(DEV)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    L = mesh.UniformLaplacian(V, faces)
    y = L @ x
    y.backward(g)
    torch.cuda.synchronize()
    # beyond the caller's x and g, the product y and the gradient x.grad (4 x 252 MB) are the only big tensors
    extra = torch.cuda.max_memory_allocated() - base - 2 * x.numel() * 4
    assert extra < 512 * 2 ** 20, extra
    rows = np.sort(np.random.default_rng(0).choice(V, 4096, replace=False))
    # the oracle on the faces around the sampled rows and their neighbours: exact for the rows and the
    # neighbours' degrees, which weight the backward
    t = M.topology(V, faces_np[np.isin(faces_np, rows).any(1)])
    t = M.topology(V, faces_np[np.isin(faces_np, np.unique(t["adj"])).any(1)])
    xs, gs = x.detach().cpu().numpy().astype(np.float64), g.cpu().numpy().astype(np.float64)
    yh, gh = y.detach().cpu().numpy(), x.grad.cpu().numpy()
    w = t["weight"].astype(np.float64)
    tol_y, tol_g = 1e-6 * np.abs(xs).max(), 1e-6 * np.abs(gs).max()
    for i in rows:
        nb = t["adj"][t["adj_ptr"][i]:t["adj_ptr"][i + 1]]
        nb = nb[nb != i]
        ref_y = w[i] * xs[:, nb].sum(1) - xs[:, i]
        ref_g = (w[nb][None, :, None] * gs[:, nb]).sum(1) - gs[:, i]
        assert np.abs(yh[:, i] - ref_y).max() <= tol_y
        assert np.abs(gh[:, i] - ref_g).max() <= tol_g


def test_tutorial_step_matches_the_dense_laplacian():
    """prepare_vertices -> dibr_rasterization -> texture_mapping -> L1 + mask_iou + Laplacian, backward:
    UniformLaplacian in place of the dense uniform_laplacian changes the gradients by < 1e-5 of scale."""
    verts, f = synthetic.icosphere(3)
    V, faces = len(verts), T(np.asarray(f, np.int64))
    rng = np.random.default_rng(4)
    v0 = T(verts.astype(np.float32))
    v_init = (verts * (1 + 0.05 * rng.uniform(-1, 1, (V, 1)))).astype(np.float32)[None]
    proj = T(np.array([[1 / math.tan(math.pi / 8)], [1 / math.tan(math.pi / 8)], [-1.]], np.float32))
    Tm = T(np.array([[[1, 0, 0], [0, 1, 0], [0, 0, 1], [0, 0, -3]]], np.float32))
    uvs = T(rng.uniform(0, 1, (1, len(f), 3, 2)).astype(np.float32))
    tex0 = rng.uniform(0, 1, (1, 3, 64, 64)).astype(np.float32)
    target = T(rng.uniform(0, 1, (1, 128, 128, 3)).astype(np.float32))
    target_mask = T((rng.uniform(0, 1, (1, 128, 128)) > 0.5).astype(np.float32))

    def step(lap):
        v = T(v_init, True)
        tex = T(tex0, True)
        fvc, fvi, fn = prepare_vertices(v, faces, proj, camera_transform=Tm)
        uv, soft, idx = dibr_rasterization(128, 128, fvc[..., 2], fvi, uvs, fn[..., 2])
        img = texture_mapping(uv, tex, mode="bilinear")
        loss = (img - target).abs().mean() + mask_iou(soft, target_mask) + (lap(v[0] - v0) ** 2).mean() * V * 3
        loss.backward()
        return v.grad, tex.grad

    Ls = mesh.UniformLaplacian(V, faces)
    Ld = mesh.uniform_laplacian(V, faces)
    gv, gt = step(lambda d: Ls @ d)
    rv, rt = step(lambda d: torch.matmul(Ld, d))
    assert float((gv - rv).abs().max()) <= 1e-5 * float(rv.abs().max())
    assert float((gt - rt).abs().max()) <= 1e-5 * float(rt.abs().max())


def test_workspace_at_an_odd_address(monkeypatch):
    """Every workspace starting at byte 1 of a larger buffer: the outputs of an aligned one."""
    V, f = synthetic.icosphere(3)
    faces_np = np.concatenate([np.asarray(f), fan(300)[1]])            # a long row among short ones
    V = max(len(V), 302)
    faces = T(faces_np)
    x = torch.randn((2, V, 3), generator=torch.Generator(device="cpu").manual_seed(2)).to(DEV)

    def run():
        L = mesh.UniformLaplacian(V, faces)
        return [L @ x, L.to_dense(), mesh.adjacency_matrix(V, faces)._indices()]

    want = run()
    scratch, odd = _lib.scratch, []
    monkeypatch.setattr(_lib, "scratch", lambda n, device: odd.append(n) or scratch(int(n) + 1, device)[1:])
    got = run()
    assert odd
    for a, b in zip(want, got):
        assert torch.equal(a, b)
