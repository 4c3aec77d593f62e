"""Marching tetrahedra and subdivide_tetmesh on sm_90a (csrc/mesh_topology.cu) against the reference's
own outputs (tests/golden/marching_tets.npz) and the fp64 torch restatement (oracle/marching_tets.py):
vertices, faces and tet indices equal to the reference's, gradients within 1e-6 of scale; the
Freudenthal grid against fp64; the reference's quirks and this library's deviations; determinism; one
synchronising read per call and none in the backward; a resolution-128 grid in bounded memory; and
one DMTet tutorial step."""
import os
import warnings

import numpy as np
import pytest
import torch

from kaolin_b200 import _lib, synthetic
from kaolin_b200.ops import conversions, mesh
from oracle import marching_tets as O
from oracle import subdivision as OS

pytestmark = pytest.mark.gpu
DEV = "cuda"
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "marching_tets.npz"))
MT_CASES = [str(c) for c in G["mt_cases"]]
SUB_CASES = [str(c) for c in G["sub_cases"]]
TABLE = O.case_table(G["single_0123_out_faces"], G["single_0123_nf"])
T_ = lambda a, grad=False: torch.from_numpy(np.ascontiguousarray(a)).to(DEV).requires_grad_(grad)
EPS = 2.0 ** -24


def traced(fn):
    _lib.trace_begin()
    try:
        out = fn()
    finally:
        ran = [name for name, _ in _lib.trace_end(1024)]
    return out, ran


def as_np(a):
    return a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


def rel(a, ref, scale):
    """Largest difference over scale; NaN and infinite positions must be equal."""
    a, ref = np.asarray(as_np(a), np.float64), np.asarray(as_np(ref), np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(ref)), "NaN positions differ"
    inf = np.isinf(ref)
    assert np.array_equal(a[inf], ref[inf]) and np.array_equal(np.isinf(a), inf), "infinities differ"
    ok = ~np.isnan(ref) & ~inf
    return float(np.abs(a[ok] - ref[ok]).max(initial=0)) / max(float(scale), 1e-30)


def finite_max(a):
    a = np.abs(np.asarray(as_np(a), np.float64))
    return float(a[np.isfinite(a)].max(initial=0.0))


def run(verts, tets, sdf, w=None, return_tet_idx=True, build_once=False):
    """Ours with autograd -> (per-view outputs, grad_vertices, grad_sdf)."""
    v = verts.detach().clone().requires_grad_(True)
    s = sdf.detach().clone().requires_grad_(True)
    if build_once:
        out = conversions.MarchingTetrahedra(v.shape[1], tets)(v, s, return_tet_idx)
    else:
        out = conversions.marching_tetrahedra(v, tets, s, return_tet_idx)
    if w is not None:
        flat = torch.cat(out[0])
        if flat.numel():
            (flat * w).sum().backward()
    return out, v.grad, s.grad


def oracle(verts, tets, sdf, w=None, dtype=torch.float64):
    v = verts.detach().to(dtype).clone().requires_grad_(True)
    s = sdf.detach().to(dtype).clone().requires_grad_(True)
    out = O.marching(v, as_np(tets), s, TABLE)
    if w is not None:
        flat = torch.cat([o[0] for o in out])
        if flat.numel():
            (flat * w.to(dtype)).sum().backward()
    return out, v.grad, s.grad


@pytest.mark.parametrize("build_once", [False, True])
@pytest.mark.parametrize("case", MT_CASES)
def test_against_the_reference(case, build_once):
    verts, tets, sdf = T_(G[f"{case}_vertices"]), T_(G[f"{case}_tets"]), T_(G[f"{case}_sdf"])
    w = T_(G[f"{case}_w"])
    (out, gv, gs), ran = traced(lambda: run(verts, tets, sdf, w, build_once=build_once))
    assert isinstance(out, list) and len(out) == 3 and all(len(o) == verts.shape[0] for o in out)
    assert [len(o) for o in out[0]] == list(G[f"{case}_nv"]) and [len(o) for o in out[1]] == list(G[f"{case}_nf"])
    assert "mt_classify_kernel" in ran and "tet_edges_kernel" in ran
    flat = torch.cat(out[0]).detach().cpu().numpy()
    assert np.array_equal(flat, G[f"{case}_out_vertices"], equal_nan=True)         # bit-equal, NaNs included
    num = ~np.isnan(flat)                 # zeros keep their sign; a NaN's sign bit is the platform's
    assert np.array_equal(np.signbit(flat[num]), np.signbit(G[f"{case}_out_vertices"][num]))
    faces, tet_idx = torch.cat(out[1]), torch.cat(out[2])
    assert faces.dtype == torch.int64 and tet_idx.dtype == torch.int64
    assert torch.equal(faces.cpu(), torch.from_numpy(G[f"{case}_out_faces"].astype(np.int64)))
    assert torch.equal(tet_idx.cpu(), torch.from_numpy(G[f"{case}_tet_idx"].astype(np.int64)))
    if flat.size:
        # only the reference's index_add order differs
        assert rel(gv, G[f"{case}_grad_vertices"], finite_max(G[f"{case}_grad_vertices"])) <= 1e-6
        assert rel(gs, G[f"{case}_grad_sdf"], finite_max(G[f"{case}_grad_sdf"])) <= 1e-6


def test_return_tet_idx_false_gives_two_lists():
    case = "cube"
    verts, tets, sdf = T_(G[f"{case}_vertices"]), T_(G[f"{case}_tets"]), T_(G[f"{case}_sdf"])
    out = conversions.marching_tetrahedra(verts, tets, sdf)
    assert len(out) == 2 and all(isinstance(o, tuple) and len(o) == 4 for o in out)
    assert torch.equal(torch.cat(out[1]).cpu(), torch.from_numpy(G[f"{case}_out_faces"].astype(np.int64)))


def run_sub(verts, tets, feats, w, wf):
    v = verts.detach().clone().requires_grad_(True)
    f = None if feats is None else feats.detach().clone().requires_grad_(True)
    out = mesh.subdivide_tetmesh(v, tets, f)
    loss = (out[0] * w).sum() + (0 if f is None else (out[2] * wf).sum())
    loss.backward()
    return out, v.grad, None if f is None else f.grad


@pytest.mark.parametrize("case", SUB_CASES)
def test_subdivide_against_the_reference(case):
    feats = T_(G[f"{case}_features"]) if f"{case}_features" in G else None
    wf = T_(G[f"{case}_wf"]) if feats is not None else None
    (out, gv, gf), ran = traced(lambda: run_sub(T_(G[f"{case}_vertices"]), T_(G[f"{case}_tets"]), feats,
                                                T_(G[f"{case}_w"]), wf))
    # the trace sees this thread's launches: the build and the forward (autograd runs the backward elsewhere)
    assert "tet_edges_kernel" in ran and "tet_subdivide_forward_kernel" in ran and "tet_children_kernel" in ran
    assert len(out) == (2 if feats is None else 3)
    assert out[1].dtype == torch.int64
    assert torch.equal(out[1].cpu(), torch.from_numpy(G[f"{case}_out_tets"].astype(np.int64)))
    assert rel(out[0], G[f"{case}_out_vertices"], finite_max(G[f"{case}_vertices"])) <= 1e-7
    assert rel(gv, G[f"{case}_grad_vertices"], finite_max(G[f"{case}_grad_vertices"])) <= 1e-6
    if feats is not None:
        assert rel(out[2], G[f"{case}_out_features"], finite_max(G[f"{case}_features"])) <= 1e-7
        assert rel(gf, G[f"{case}_grad_features"], finite_max(G[f"{case}_grad_features"])) <= 1e-6


def grid(res, seed):
    """The Freudenthal grid with every tet's corners randomly permuted."""
    verts, tets = synthetic.freudenthal_grid(res)
    rng = np.random.default_rng(seed)
    tets = np.take_along_axis(tets, np.argsort(rng.random(tets.shape), 1), 1)
    return verts, tets


def sphere_sdf(verts, B, seed, noise=0.02):
    """A noisy sphere of radius ~0.3 per view, with jittered vertex positions."""
    gen = torch.Generator(device="cpu").manual_seed(seed)
    v = torch.from_numpy(verts)[None] + 0.004 * (torch.rand((B,) + verts.shape, generator=gen) - 0.5)
    r = 0.25 + 0.1 * torch.rand((B, 1), generator=gen)
    s = v.norm(dim=-1) - r + noise * torch.randn(v.shape[:2], generator=gen)
    return v.to(DEV), s.to(DEV)


@pytest.mark.parametrize("res", [32, 64])
@pytest.mark.parametrize("B", [1, 4])
def test_against_fp64_on_the_freudenthal_grid(res, B):
    verts, tets_np = grid(res, res + B)
    v, s = sphere_sdf(verts, B, res * 10 + B)
    tets = T_(tets_np)
    M = conversions.MarchingTetrahedra(len(verts), tets)
    out = M(v, s, True)
    nv = sum(len(o) for o in out[0])
    w = torch.randn((nv, 3), generator=torch.Generator(device="cpu").manual_seed(B)).to(DEV)
    ours, gv, gs = run(v, tets, s, w, build_once=True)
    ref, rgv, rgs = oracle(v, tets, s, w)
    for b in range(B):
        assert torch.equal(ours[1][b].cpu(), ref[b][1]) and torch.equal(ours[2][b].cpu(), ref[b][2])
        assert torch.equal(ours[0][b], out[0][b])
        # no cancellation: s_a and -s_b have the same sign, so each step errs by half an ulp
        assert float((ours[0][b].detach().double() - ref[b][0].detach()).abs().max()) <= 4 * EPS * float(v.abs().max())
    assert rel(gv, rgv, finite_max(rgv)) <= 1e-5
    assert rel(gs, rgs, finite_max(rgs)) <= 1e-5


@pytest.mark.parametrize("res", [32, 64])
@pytest.mark.parametrize("B", [1, 4])
def test_subdivide_against_fp64_on_the_freudenthal_grid(res, B):
    verts, tets_np = grid(res, res + 7 * B)
    v, s = sphere_sdf(verts, B, res + B)
    gen = torch.Generator(device="cpu").manual_seed(res * B)
    feats = torch.cat([s[..., None], torch.randn((B, len(verts), 3), generator=gen).to(DEV)], -1)
    tets = T_(tets_np)
    y, ty, yf = mesh.subdivide_tetmesh(v, tets, feats)
    w, wf = torch.randn(y.shape, generator=gen).to(DEV), torch.randn(yf.shape, generator=gen).to(DEV)
    (out, ot, of), gv, gf = run_sub(v, tets, feats, w, wf)
    assert torch.equal(out, y) and torch.equal(of, yf) and torch.equal(ot, ty)
    vd, fd = v.double().requires_grad_(True), feats.double().requires_grad_(True)
    ry, rt, rf = O.subdivide(vd, tets_np, fd)
    ((ry * w.double()).sum() + (rf * wf.double()).sum()).backward()
    assert torch.equal(ot.cpu(), rt)
    assert float((out.double() - ry).abs().max()) <= EPS * float(v.abs().max())
    assert float((of.double() - rf).abs().max()) <= EPS * float(feats.abs().max())
    # an input row sums its own weight and a half of each of its at most 14 edges' (the grid's degree):
    # at most 16 terms of total weight <= 8 |w|, summed in fp32
    deg = int(np.bincount(np.unique(np.sort(tets_np[:, O.PAIRS], -1).reshape(-1, 2), axis=0).ravel()).max())
    assert deg <= 14
    assert float((gv.double() - vd.grad).abs().max()) <= 16 * EPS * 8 * float(w.abs().max())
    assert float((gf.double() - fd.grad).abs().max()) <= 16 * EPS * 8 * float(wf.abs().max())


def test_zero_and_nan_sdf_count_as_outside():
    verts = T_(np.array([[[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]]], np.float32))
    tets = T_(np.array([[0, 1, 2, 3]]))
    for vals, nv in (([0, 0, 0, 0], 0), ([float("nan")] * 4, 0), ([1, 0, 0, 0], 3), ([1, float("nan"), 0, -1], 3),
                     ([1, 1, 1, 1], 0)):
        out = conversions.marching_tetrahedra(verts, tets, T_(np.array([vals], np.float32)))
        assert len(out[0][0]) == nv and out[0][0].shape == (nv, 3) and out[1][0].shape == (nv // 3, 3)
    # a NaN sdf on a sign-change edge gives a NaN vertex, as in the reference
    out = conversions.marching_tetrahedra(verts, tets, T_(np.array([[float("nan"), 1, 1, 1]], np.float32)))
    assert bool(torch.isnan(out[0][0]).all())


def test_degenerate_tets_keep_their_degenerate_faces():
    verts = T_(np.random.default_rng(0).normal(size=(1, 4, 3)).astype(np.float32))
    tets = T_(np.array([[0, 0, 1, 2], [0, 1, 2, 3]]))
    sdf = T_(np.array([[1, -1, -1, -1]], np.float32))
    out = conversions.marching_tetrahedra(verts, tets, sdf, True)
    ref = O.marching(verts, as_np(tets), sdf, TABLE)[0]
    assert torch.equal(out[1][0].cpu(), ref[1]) and torch.equal(out[2][0].cpu(), ref[2])
    f = out[1][0]
    assert bool((f[:, 0] == f[:, 1]).any() | (f[:, 1] == f[:, 2]).any() | (f[:, 0] == f[:, 2]).any())


def test_empty_inputs():
    verts = torch.rand((2, 4, 3), device=DEV)
    sdf = torch.rand((2, 4), device=DEV) - 0.5
    assert conversions.marching_tetrahedra(verts[:0], T_(np.array([[0, 1, 2, 3]])), sdf[:0]) == []
    no_tets = T_(np.zeros((0, 4), np.int64))
    for tets, s in ((no_tets, sdf), (T_(np.array([[0, 1, 2, 3]])), sdf.abs() + 1)):
        x = verts.clone().requires_grad_(True)
        v, f, t = conversions.marching_tetrahedra(x, tets, s, True)
        assert len(v) == 2 and all(a.shape == (0, 3) and b.shape == (0, 3) and c.shape == (0,)
                                   for a, b, c in zip(v, f, t))
        assert v[0].dtype == torch.float32 and f[0].dtype == torch.int64 and t[0].dtype == torch.int64
        torch.cat(v).sum().backward()
        assert bool((x.grad == 0).all())
    y, t = mesh.subdivide_tetmesh(verts, no_tets)
    assert torch.equal(y, verts) and t.shape == (0, 4)


def test_non_contiguous_inputs_are_served():
    verts, tets_np = grid(8, 1)
    v, s = sphere_sdf(verts, 2, 2)
    pred = torch.cat([s[..., None], torch.rand_like(s)[..., None]], -1)          # (B, V, 2): pred[..., 0]
    tets = T_(tets_np)
    a = conversions.marching_tetrahedra(v.transpose(1, 2).contiguous().transpose(1, 2), tets, pred[..., 0], True)
    b = conversions.marching_tetrahedra(v, tets, s.contiguous(), True)
    for x, y in zip(a, b):
        assert all(torch.equal(p, q) for p, q in zip(x, y))
    tets_nc = torch.cat([tets, tets], 1)[:, :4]
    assert not tets_nc.is_contiguous()
    c = conversions.marching_tetrahedra(v, tets_nc, s, True)
    assert all(torch.equal(p, q) for x, y in zip(b, c) for p, q in zip(x, y))


def test_deviations_raise():
    verts = torch.rand((1, 4, 3), device=DEV)
    sdf = torch.rand((1, 4), device=DEV)
    tets = T_(np.array([[0, 1, 2, 3]]))
    for call in (lambda: conversions.marching_tetrahedra(verts.double(), tets, sdf),
                 lambda: conversions.marching_tetrahedra(verts, tets, sdf.double()),
                 lambda: conversions.marching_tetrahedra(verts.half(), tets, sdf),
                 lambda: conversions.marching_tetrahedra(verts, tets.int(), sdf),
                 lambda: mesh.subdivide_tetmesh(verts.double(), tets),
                 lambda: mesh.subdivide_tetmesh(verts, tets.int()),
                 lambda: mesh.subdivide_tetmesh(verts, tets, torch.rand((1, 4, 2), device=DEV).double())):
        with pytest.raises(RuntimeError, match="not implemented"):
            call()
    for bad in ([[0, 1, 2, 4]], [[0, -1, 2, 3]], [[0, 1, 2, 3], [1, 2, 3, 1 << 40]]):
        with pytest.raises(IndexError):
            conversions.marching_tetrahedra(verts, T_(np.array(bad)), sdf)
        with pytest.raises(IndexError):
            conversions.MarchingTetrahedra(4, T_(np.array(bad)))
        with pytest.raises(IndexError):
            mesh.subdivide_tetmesh(verts, T_(np.array(bad)))
    with pytest.raises(RuntimeError, match="tets"):
        conversions.MarchingTetrahedra(4, T_(np.array([[0, 1, 2]])))
    with pytest.raises(RuntimeError, match="sdf"):
        conversions.MarchingTetrahedra(4, tets)(verts, sdf[:, :3])


def test_runs_are_byte_identical():
    verts, tets_np = grid(24, 3)
    v, s = sphere_sdf(verts, 3, 4)
    feats = torch.randn((3, len(verts), 2), device=DEV)
    tets = T_(tets_np)

    def once():
        x, sd = v.clone().requires_grad_(True), s.clone().requires_grad_(True)
        verts_out, faces, tet_idx = conversions.MarchingTetrahedra(len(verts), tets)(x, sd, True)
        flat = torch.cat(verts_out)
        flat.backward(torch.cos(torch.arange(flat.numel(), device=DEV, dtype=torch.float32)).view_as(flat))
        xf, ff = v.clone().requires_grad_(True), feats.clone().requires_grad_(True)
        y, t, yf = mesh.subdivide_tetmesh(xf, tets, ff)
        (y.sin().sum() + yf.cos().sum()).backward()
        return [flat.detach(), torch.cat(faces), torch.cat(tet_idx), x.grad, sd.grad, y.detach(), t, yf.detach(),
                xf.grad, ff.grad]

    for p, q in zip(once(), once()):
        assert torch.equal(p.view(torch.uint8) if p.is_floating_point() else p,
                           q.view(torch.uint8) if q.is_floating_point() else q)


def test_one_synchronising_read_per_call_and_none_in_the_backward():
    verts, tets_np = grid(16, 5)
    v, s = sphere_sdf(verts, 2, 6)
    M = conversions.MarchingTetrahedra(len(verts), T_(tets_np))
    x, sd = v.clone().requires_grad_(True), s.clone().requires_grad_(True)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = M(x, sd, True)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [w for w in caught if "called a synchronizing" in str(w.message)]
    assert len(syncs) == 1, [str(w.message) for w in caught]
    flat = torch.cat(out[0])
    g = torch.randn_like(flat)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        flat.backward(g)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    xr, sr = v.clone().requires_grad_(True), s.clone().requires_grad_(True)
    ref = conversions.marching_tetrahedra(xr, T_(tets_np), sr, True)
    torch.cat(ref[0]).backward(g)
    assert torch.equal(x.grad, xr.grad) and torch.equal(sd.grad, sr.grad)


def test_resolution_128_in_bounded_memory():
    verts, tets_np = synthetic.freudenthal_grid(128)
    V, T = len(verts), len(tets_np)
    assert T == 6 * 128 ** 3
    tets = T_(tets_np)
    v, s = sphere_sdf(verts, 1, 128, noise=0.0)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    M = conversions.MarchingTetrahedra(V, tets)
    torch.cuda.synchronize()
    E = M._topo.num_edges
    # the build: workspace (count, long rows, corner CSR, degree, weight, edge offsets: 6 V ints; raw
    # neighbours 12 T, corners 4 T) and the capacity-sized outputs (adjacency and its edge ids 12 T each,
    # edges 12 T, tet_edge 6 T, offsets V), then the trimmed copies (<= 2 * 2E + 2E ints)
    build_bound = 4 * (7 * V + 16 * T + 42 * T + 6 * E) + (64 << 20)
    assert torch.cuda.max_memory_allocated() - base <= build_bound
    held = torch.cuda.memory_allocated() - base
    assert held <= 4 * (V + 6 * T + 6 * E) + (8 << 20)        # adj_ptr, tet_edge, adjacency, edge ids, edges
    x, sd = v.clone().requires_grad_(True), s.clone().requires_grad_(True)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = M(x, sd, True)
    nv, nf = len(out[0][0]), len(out[1][0])
    out[0][0].backward(torch.ones_like(out[0][0]))
    torch.cuda.synchronize()
    # flags and their scan (2 (E + 2T) ints), vid (E ints), the outputs (vertices, faces, tet_idx), the
    # gradient of the output and of x and sdf
    call_bound = 4 * (2 * (E + 2 * T) + E) + 12 * nv + 32 * nf + 12 * nv + 16 * V + (64 << 20)
    assert torch.cuda.max_memory_allocated() - base <= call_bound
    # a closed sphere's surface: every edge in exactly two faces, and no degenerate face
    f = out[1][0]
    assert nf > 0 and int(f.min()) >= 0 and int(f.max()) == nv - 1
    assert bool(((f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])).all())
    e = torch.sort(torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1).values
    _, counts = torch.unique(e[:, 0] * nv + e[:, 1], return_counts=True)
    assert bool((counts == 2).all())
    assert bool(torch.isfinite(x.grad).all()) and bool(torch.isfinite(sd.grad).all())


def laplace_regularizer(verts, faces):
    """The DMTet tutorial's regulariser: mean over vertices of |sum over incident face corners of the
    two edge vectors / max(2 * corners, 1)|^2."""
    term = torch.zeros_like(verts)
    norm = torch.zeros_like(verts[:, :1])
    for k in range(3):
        v0, v1, v2 = (verts[faces[:, (k + u) % 3]] for u in range(3))
        term = term.index_add(0, faces[:, k], (v1 - v0) + (v2 - v0))
        norm = norm.index_add(0, faces[:, k], torch.full_like(v0[:, :1], 2.0))
    return ((term / norm.clamp(min=1.0)) ** 2).mean()


def test_dmtet_tutorial_step_matches_the_oracle():
    """A learnable (V, 4) prediction on a resolution-32 grid (sdf = pred[:, 0], deformation =
    pred[:, 1:]) -> MarchingTetrahedra -> subdivide_trianglemesh(, 1) -> the tutorial's Laplacian
    regulariser plus sum(verts * w), backward: against the same step through the fp64 oracles."""
    res = 32
    verts_np, tets_np = grid(res, 9)
    tets = T_(tets_np)
    base = T_(verts_np)
    V = len(verts_np)
    gen = torch.Generator(device="cpu").manual_seed(10)
    init = torch.cat([(base.cpu().norm(dim=-1, keepdim=True) - 0.3 + 0.02 * torch.randn((V, 1), generator=gen)),
                      0.5 * torch.randn((V, 3), generator=gen)], -1).to(DEV)
    M = conversions.MarchingTetrahedra(V, tets)

    def step(dtype, march, subdivide):
        pred = init.to(dtype).clone().requires_grad_(True)
        sdf, deform = pred[:, 0], pred[:, 1:]
        verts = (base.to(dtype) + torch.tanh(deform) / res).unsqueeze(0)
        mv, mf = march(verts, sdf.unsqueeze(0))
        fine, ff = subdivide(mv.unsqueeze(0), mf)
        w = torch.cos(torch.arange(fine.numel(), device=DEV, dtype=dtype)).view_as(fine)
        loss = laplace_regularizer(fine[0], ff) + (fine * w).sum()
        loss.backward()
        return pred.grad, ff

    def ours_march(v, s):
        out = M(v, s)
        return out[0][0], out[1][0]

    def oracle_march(v, s):
        out = O.marching(v, tets_np, s, TABLE)[0]
        return out[0], out[1].to(DEV)

    def oracle_subdivide(v, f):
        y, fine_faces = OS.subdivide(v, f.cpu().numpy(), 1)
        return y, fine_faces.to(DEV)

    g, ff = step(torch.float32, ours_march, lambda v, f: mesh.subdivide_trianglemesh(v, f, 1))
    rg, rff = step(torch.float64, oracle_march, oracle_subdivide)
    assert torch.equal(ff, rff)
    for k in (slice(0, 1), slice(1, 4)):          # the sdf and the deformation
        assert float((g[:, k].double() - rg[:, k]).abs().max()) <= 1e-5 * float(rg[:, k].abs().max())


def test_workspace_at_an_odd_address(monkeypatch):
    """Every workspace starting at byte 1 of a larger buffer: the outputs of an aligned one."""
    verts, tets_np = grid(16, 3)
    v, s = sphere_sdf(verts, 3, 4)
    feats = torch.randn((3, len(verts), 2), device=DEV)
    tets = T_(tets_np)

    def run():
        verts_out, faces, tet_idx = conversions.MarchingTetrahedra(len(verts), tets)(v, s, True)
        return [torch.cat(verts_out), torch.cat(faces), torch.cat(tet_idx), *mesh.subdivide_tetmesh(v, tets, feats)]

    want = run()
    scratch, odd = _lib.scratch, []
    monkeypatch.setattr(_lib, "scratch", lambda n, device: odd.append(n) or scratch(int(n) + 1, device)[1:])
    got = run()
    assert odd
    for a, b in zip(want, got):
        assert torch.equal(a, b)
