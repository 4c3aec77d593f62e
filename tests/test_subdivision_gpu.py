"""Loop subdivision on sm_90a (csrc/mesh_topology.cu) against the reference's own outputs
(tests/golden/subdivision.npz) and the fp64 torch restatement (oracle/subdivision.py): faces exact,
vertices and gradients within 1e-6 of scale of the goldens and within a rounding bound of fp64; the
reference's quirks and this library's deviations; determinism; no host synchronisation; c5's face count;
and one DIB-R tutorial step with a learnable alpha."""
import math
import os

import numpy as np
import pytest
import torch

from kaolin_b200 import _lib, synthetic
from kaolin_b200.metrics.render import mask_iou
from kaolin_b200.ops import mesh
from kaolin_b200.render.mesh import dibr_rasterization, prepare_vertices, texture_mapping
from oracle import subdivision as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "subdivision.npz"))
CASES = [str(c) for c in G["cases"]]
T = lambda a, grad=False: torch.from_numpy(np.ascontiguousarray(a)).to(DEV).requires_grad_(grad)
EPS = 2.0 ** -24


def traced(fn):
    _lib.trace_begin()
    try:
        out = fn()
    finally:
        ran = [name for name, _ in _lib.trace_end(1024)]
    return out, ran


def rel(a, ref, scale):
    """Largest difference over scale; NaN positions must be equal."""
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    ref = ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else ref
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(ref)), "NaN positions differ"
    ok = ~np.isnan(ref)
    return float(np.abs(a[ok] - ref[ok]).max(initial=0)) / max(float(scale), 1e-30)


def nanmax_abs(a):
    return float(np.nanmax(np.abs(np.asarray(a, np.float64)), initial=0.0))


def fan(n):
    """One vertex in n triangles (0, i+1, i+2): degree n + 1, an open boundary."""
    return n + 2, np.stack([np.zeros(n, np.int64), np.arange(1, n + 1), np.arange(2, n + 2)], 1)


def run(verts, faces, iterations, alpha, w):
    """Ours, with autograd: -> out, faces, grad_vertices, grad_alpha (or None)."""
    v = verts.detach().clone().requires_grad_(True)
    a = None if alpha is None else alpha.detach().clone().requires_grad_(True)
    out, f = mesh.subdivide_trianglemesh(v, faces, iterations, a)
    (out * w).sum().backward()
    return out.detach(), f, v.grad, None if a is None else a.grad


def oracle(verts, faces, iterations, alpha, w):
    """The fp64 restatement on the GPU, with autograd."""
    v = verts.detach().double().clone().requires_grad_(True)
    a = None if alpha is None else alpha.detach().double().clone().requires_grad_(True)
    out, f = O.subdivide(v, faces.cpu().numpy(), iterations, a)
    (out * w.double()).sum().backward()
    return out.detach(), f, v.grad, None if a is None else a.grad


@pytest.mark.parametrize("case", CASES)
def test_against_the_reference(case):
    verts, faces, it = T(G[f"{case}_vertices"]), T(G[f"{case}_faces"]), int(G[f"{case}_iterations"])
    alpha = T(G[f"{case}_alpha"]) if f"{case}_alpha" in G else None
    w = T(G[f"{case}_w"])
    ((out, f, gv, ga), ran) = traced(lambda: run(verts, faces, it, alpha, w))
    assert torch.equal(f.cpu(), torch.from_numpy(G[f"{case}_out_faces"].astype(np.int64)))
    assert f.dtype == torch.int64 and out.shape == G[f"{case}_out"].shape
    if len(G[f"{case}_faces"]):          # the trace sees this thread's launches: the build and the forward
        assert "subdiv_edges_kernel" in ran and "subdiv_forward_kernel" + ("<alpha>" if alpha is not None else "") in ran
    assert rel(out, G[f"{case}_out"], nanmax_abs(G[f"{case}_vertices"])) <= 1e-6
    assert rel(gv, G[f"{case}_grad_vertices"], nanmax_abs(G[f"{case}_grad_vertices"])) <= 1e-6
    if alpha is not None:
        # (g . s) / n - g . x: the two dot products nearly cancel on a smooth surface, and the reference's
        # fp32 result is itself up to 1e-5 of its largest value from exact arithmetic; the scale is the
        # size of the terms that cancel
        scale = nanmax_abs(G[f"{case}_w"]) * nanmax_abs(G[f"{case}_vertices"])
        assert rel(ga, G[f"{case}_grad_alpha"], scale) <= 1e-6


def test_reference_tests_expected_tensors():
    v, f = T(G["ref_vertices"]), T(G["ref_faces"])
    for alpha, key in ((None, "ref_expected_default"), (torch.zeros((1, 12), device=DEV), "ref_expected_zero_alpha")):
        out, faces = mesh.subdivide_trianglemesh(v, f, 1, alpha)
        assert torch.equal(faces.cpu(), torch.from_numpy(G["ref_expected_faces"]))
        assert float((out.cpu() - torch.from_numpy(G[key])).abs().max()) <= 1e-4
    out, faces = mesh.subdivide_trianglemesh(v, f, 5)
    assert faces.shape[0] == int(G["ref_5iter_faces"]) == 20 * 4 ** 5
    tri = out[0][faces]
    area = torch.linalg.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]).norm(dim=-1).sum() / 2
    assert abs(float(area) - float(G["ref_5iter_area"])) <= 1e-4


def _levels(V, faces_np, iterations):
    levels = []
    for _ in range(iterations):
        levels.append(O.level(V, faces_np))
        V, faces_np = V + len(levels[-1]["edges"]), levels[-1]["new_faces"]
    return levels


def _value_bound(levels, scale):
    """(deg + 2) * 2^-24 * scale per level, summed over the levels, with each level's largest degree."""
    return sum(int(lv["degree"].max(initial=0)) + 2 for lv in levels) * EPS * scale


def _terms(levels):
    """Terms a gradient row gathers per level: itself, deg neighbours, deg endpoints, 3 edges per corner."""
    return sum(3 + 2 * int(lv["degree"].max(initial=0)) + 3 * int(np.bincount(lv["faces"].ravel()).max(initial=0))
               for lv in levels)


def _grad_bounds(x, faces, iterations, alpha, w, levels):
    """Per-element bounds of the vertex and alpha gradients: every weight of the transposed stencils is
    >= 0 (alpha in [0, 1]), so the fp64 gradient of sum(out * |w|) is the sum of the magnitudes of the
    terms each gradient row adds, and fp32 summation of n terms errs by at most n * 2^-24 times that."""
    _, _, mag, _ = oracle(x, faces, iterations, alpha, w.abs())
    t = _terms(levels)
    gv = t * EPS * mag
    # alpha: (g . s) / n - g . x and the carried alpha's stencils; terms of at most 3 |g| |x| each
    ga = t * EPS * 6 * float(x.abs().max()) * float(mag.abs().max())
    return gv, ga


@pytest.mark.parametrize("level", [4, 5])
@pytest.mark.parametrize("iterations", [1, 2, 3])
@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("learn_alpha", [False, True])
def test_against_fp64(level, iterations, B, learn_alpha):
    verts, f = synthetic.icosphere(level)
    faces_np = np.asarray(f, np.int64)
    V = len(verts)
    gen = torch.Generator(device="cpu").manual_seed(level * 10 + iterations)
    x = (torch.from_numpy(np.asarray(verts, np.float32))[None] * (1 + 0.1 * torch.rand((B, V, 1), generator=gen))).to(DEV)
    alpha = torch.rand((B, V), generator=gen).to(DEV) if learn_alpha else None
    faces = T(faces_np)
    S = mesh.LoopSubdivision(V, faces, iterations)
    w = torch.randn((B, S.num_output_vertices, 3), generator=gen).to(DEV)
    out, fo, gv, ga = run(x, faces, iterations, alpha, w)
    ro, rf, rgv, rga = oracle(x, faces, iterations, alpha, w)
    assert torch.equal(fo.cpu(), rf)
    levels = _levels(V, faces_np, iterations)
    assert float((out.double() - ro).abs().max()) <= _value_bound(levels, float(x.abs().max()))
    bv, ba = _grad_bounds(x, faces, iterations, alpha, w, levels)
    assert bool(((gv.double() - rgv).abs() <= bv).all())
    if learn_alpha:
        assert float((ga.double() - rga).abs().max()) <= ba


def test_fan_vertex_in_10000_triangles():
    V, faces_np = fan(10000)
    gen = torch.Generator(device="cpu").manual_seed(3)
    x = (torch.rand((2, V, 3), generator=gen) * 2 - 1).to(DEV)
    alpha = torch.rand((2, V), generator=gen).to(DEV)
    faces = T(faces_np)
    levels = _levels(V, faces_np, 1)
    lv = levels[0]
    assert int(lv["degree"][0]) == 10001
    deg = np.concatenate([lv["degree"], np.full(len(lv["edges"]), 6)]).astype(np.float64)
    for a in (None, alpha):
        w = torch.randn((2, V + len(lv["edges"]), 3), generator=gen).to(DEV)
        out, f, gv, ga = run(x, faces, 1, a, w)
        ro, rf, rgv, rga = oracle(x, faces, 1, a, w)
        assert torch.equal(f.cpu(), rf)
        bound = (deg + 2)[None, :, None] * EPS * float(x.abs().max())
        assert np.all(np.abs(out.double().cpu().numpy() - ro.cpu().numpy()) <= bound)
        bv, ba = _grad_bounds(x, faces, 1, a, w, levels)
        assert bool(((gv.double() - rgv).abs() <= bv).all())
        if a is not None:
            assert float((ga.double() - rga).abs().max()) <= ba


def test_unreferenced_vertex_is_nan_whatever_alpha():
    faces = T(np.array([[0, 1, 2], [0, 2, 3]]))
    x = torch.rand((2, 5, 3), device=DEV)                      # vertex 4 is in no face
    for alpha in (None, torch.zeros((2, 5), device=DEV), torch.full((2, 5), 0.5, device=DEV)):
        out, _ = mesh.subdivide_trianglemesh(x, faces, 2, alpha)
        nan_rows = torch.isnan(out).any(-1)
        assert bool(nan_rows[:, 4].all()) and int(nan_rows.sum()) == 2
        assert not bool(torch.isnan(out[:, :4]).any())


def test_no_faces_gives_all_nan():
    x = torch.rand((3, 4, 3), device=DEV)
    for alpha in (None, torch.zeros((3, 4), device=DEV)):
        out, faces = mesh.subdivide_trianglemesh(x, T(np.zeros((0, 3), np.int64)), 2, alpha)
        assert out.shape == (3, 4, 3) and bool(torch.isnan(out).all())
        assert faces.shape == (0, 3) and faces.dtype == torch.int64


def test_zero_iterations_returns_the_inputs():
    x = torch.rand((2, 3, 3), device=DEV)
    f = T(np.array([[0, 1, 2]]))
    out, faces = mesh.subdivide_trianglemesh(x, f, 0, torch.rand((2, 3), device=DEV))
    assert out is x and faces is f
    S = mesh.LoopSubdivision(3, f, 0)
    assert S(x) is x and S.faces is f


def test_gradients_carry_the_nan_pattern():
    faces = T(np.array([[0, 1, 2], [0, 2, 3]]))
    x = torch.rand((1, 5, 3), device=DEV, requires_grad=True)
    out, _ = mesh.subdivide_trianglemesh(x, faces, 1)
    out.backward(torch.ones_like(out))
    # default alpha: (1 - NaN) g at the unreferenced vertex; the others stay finite
    assert bool(torch.isnan(x.grad[0, 4]).all()) and not bool(torch.isnan(x.grad[0, :4]).any())
    x.grad = None
    a = torch.rand((1, 5), device=DEV, requires_grad=True)
    out, _ = mesh.subdivide_trianglemesh(x, faces, 1, a)
    out.backward(torch.ones_like(out))
    # given alpha: (g . s) / n = 0 / 0 for alpha; the vertex's own gradient (1 - alpha) g is finite
    assert bool(torch.isnan(a.grad[0, 4])) and not bool(torch.isnan(a.grad[0, :4]).any())
    assert not bool(torch.isnan(x.grad).any())


def test_any_batch_and_alpha_must_match_it():
    v, f = synthetic.icosphere(1)
    faces = T(np.asarray(f, np.int64))
    x = torch.rand((5, len(v), 3), device=DEV)
    a = torch.rand((5, len(v)), device=DEV)
    out, _ = mesh.subdivide_trianglemesh(x, faces, 2, a)
    for b in range(5):                                         # batched = per view
        ob, _ = mesh.subdivide_trianglemesh(x[b:b + 1], faces, 2, a[b:b + 1])
        assert torch.equal(out[b:b + 1], ob)
    with pytest.raises(RuntimeError, match="alpha"):
        mesh.subdivide_trianglemesh(x, faces, 1, a[:1])
    with pytest.raises(RuntimeError, match="alpha"):
        mesh.subdivide_trianglemesh(x, faces, 1, a[..., None])


@pytest.mark.parametrize("bad", [[[0, 1, 5]], [[0, -1, 2]], [[0, 1, 2], [3, 1, 1 << 40]]])
def test_out_of_range_index_raises(bad):
    x = torch.rand((1, 4, 3), device=DEV)
    with pytest.raises(IndexError):
        mesh.subdivide_trianglemesh(x, T(np.array(bad)), 1)
    with pytest.raises(IndexError):
        mesh.LoopSubdivision(4, T(np.array(bad)), 2)


def test_non_triangle_faces_raise():
    x = torch.rand((1, 5, 3), device=DEV)
    for bad in (np.array([[0, 1, 2, 3]]), np.array([[0, 1]]), np.array([0, 1, 2])):
        with pytest.raises(RuntimeError, match="triangle"):
            mesh.subdivide_trianglemesh(x, T(bad), 1)


def test_only_float32():
    x = torch.rand((1, 3, 3), device=DEV)
    f = T(np.array([[0, 1, 2]]))
    for call in (lambda: mesh.subdivide_trianglemesh(x.double(), f, 1),
                 lambda: mesh.subdivide_trianglemesh(x.half(), f, 1),
                 lambda: mesh.subdivide_trianglemesh(x, f, 1, torch.rand((1, 3), device=DEV).double()),
                 lambda: mesh.LoopSubdivision(3, f, 1)(x.double())):
        with pytest.raises(RuntimeError, match="not implemented"):
            call()


def test_runs_are_byte_identical():
    v, f = synthetic.icosphere(4)
    faces_np = np.concatenate([np.asarray(f, np.int64), fan(300)[1]])   # a long row among short ones
    V = max(len(v), 302)
    gen = torch.Generator(device="cpu").manual_seed(5)
    x = torch.randn((3, V, 3), generator=gen).to(DEV)
    a = torch.rand((3, V), generator=gen).to(DEV)
    faces = T(faces_np)

    def once():
        outs = []
        for alpha in (None, a):
            S = mesh.LoopSubdivision(V, faces, 2)
            xv = x.clone().requires_grad_(True)
            av = None if alpha is None else alpha.clone().requires_grad_(True)
            y = S(xv, av)
            y.backward(torch.cos(torch.arange(y.numel(), device=DEV, dtype=torch.float32)).view_as(y))
            outs += [y.detach(), S.faces, xv.grad] + ([] if av is None else [av.grad])
        return outs

    for p, q in zip(once(), once()):
        assert torch.equal(p.view(torch.uint8) if p.is_floating_point() else p,
                           q.view(torch.uint8) if q.is_floating_point() else q)


def test_loop_subdivision_makes_no_host_synchronisation():
    v, f = synthetic.icosphere(3)
    faces = T(np.asarray(f, np.int64))
    x = torch.randn((2, len(v), 3), device=DEV)
    a = torch.rand((2, len(v)), device=DEV)
    S = mesh.LoopSubdivision(len(v), faces, 2)
    g = torch.randn((2, S.num_output_vertices, 3), device=DEV)
    xs, as_ = x.clone().requires_grad_(True), a.clone().requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        y = S(xs, as_)
        y.backward(g)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    xf, af = x.clone().requires_grad_(True), a.clone().requires_grad_(True)
    yf, ff = mesh.subdivide_trianglemesh(xf, faces, 2, af)
    yf.backward(g)
    assert torch.equal(y, yf) and torch.equal(S.faces, ff)
    assert torch.equal(xs.grad, xf.grad) and torch.equal(as_.grad, af.grad)


def test_c5_face_count_in_bounded_memory():
    verts, f = synthetic.icosphere(5)
    V, faces_np = len(verts), np.asarray(f, np.int64)
    faces = T(faces_np)
    B = 8
    gen = torch.Generator(device="cpu").manual_seed(6)
    x = (torch.from_numpy(np.asarray(verts, np.float32))[None] * (1 + 0.1 * torch.rand((B, V, 1), generator=gen))).to(DEV)
    x.requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    S = mesh.LoopSubdivision(V, faces, 3)
    assert S.faces.shape == (1310720, 3)
    y = S(x)
    g = torch.randn(y.shape, generator=gen).to(DEV)
    y.backward(g)
    torch.cuda.synchronize()
    # beyond x, x.grad, y and g: the three levels' structures (about 130 MB at these sizes) and one
    # intermediate level's vertices and gradient
    extra = torch.cuda.max_memory_allocated() - base - 2 * y.numel() * 4 - 2 * x.numel() * 4
    assert extra < 256 * 2 ** 20, extra
    ro, rf, rgv, _ = oracle(x, faces, 3, None, g)
    assert torch.equal(S.faces.cpu(), rf)
    rows = torch.from_numpy(np.random.default_rng(0).choice(y.shape[1], 65536, replace=False)).to(DEV)
    levels = _levels(V, faces_np, 3)
    assert float((y.detach()[:, rows].double() - ro[:, rows]).abs().max()) <= _value_bound(levels, float(x.abs().max()))
    bv, _ = _grad_bounds(x.detach(), faces, 3, None, g, levels)
    assert bool(((x.grad.double() - rgv).abs() <= bv).all())


def test_tutorial_step_matches_the_oracle_subdivision():
    """Level-2 icosphere with a learnable alpha -> LoopSubdivision(, 2) -> prepare_vertices ->
    dibr_rasterization -> texture_mapping -> L1 + mask_iou, backward: against the same step with the
    oracle's subdivision, vertex and alpha gradients within 1e-5 of scale.  The oracle's fp32 vertices
    differ from ours in the last bits, and a silhouette pixel that changes face moves the gradients by
    more than that; so the oracle's step renders our vertices (its own plus the detached difference)
    and takes its gradients through its own subdivision."""
    verts, f = synthetic.icosphere(2)
    V, faces = len(verts), T(np.asarray(f, np.int64))
    rng = np.random.default_rng(4)
    v_init = (verts * (1 + 0.05 * rng.uniform(-1, 1, (V, 1)))).astype(np.float32)[None]
    a_init = rng.uniform(0.2, 0.8, (1, V)).astype(np.float32)
    proj = T(np.array([[1 / math.tan(math.pi / 8)], [1 / math.tan(math.pi / 8)], [-1.]], np.float32))
    Tm = T(np.array([[[1, 0, 0], [0, 1, 0], [0, 0, 1], [0, 0, -3]]], np.float32))
    S = mesh.LoopSubdivision(V, faces, 2)
    fine_faces = S.faces
    uvs = T(rng.uniform(0, 1, (1, len(fine_faces), 3, 2)).astype(np.float32))
    tex = T(rng.uniform(0, 1, (1, 3, 64, 64)).astype(np.float32))
    target = T(rng.uniform(0, 1, (1, 128, 128, 3)).astype(np.float32))
    target_mask = T((rng.uniform(0, 1, (1, 128, 128)) > 0.5).astype(np.float32))

    def step(subdivide):
        v, a = T(v_init, True), T(a_init, True)
        fine = subdivide(v, a)
        fvc, fvi, fn = prepare_vertices(fine, fine_faces, proj, camera_transform=Tm)
        uv, soft, idx = dibr_rasterization(128, 128, fvc[..., 2], fvi, uvs, fn[..., 2])
        img = texture_mapping(uv, tex, mode="bilinear")
        loss = (img - target).abs().mean() + mask_iou(soft, target_mask)
        loss.backward()
        return v.grad, a.grad

    gv, ga = step(lambda v, a: S(v, a))

    def oracle_step(v, a):
        ref = O.subdivide(v, faces.cpu().numpy(), 2, a)[0]
        return ref + (S(v.detach(), a.detach()) - ref).detach()

    rv, ra = step(oracle_step)
    assert float((gv - rv).abs().max()) <= 1e-5 * float(rv.abs().max())
    assert float((ga - ra).abs().max()) <= 1e-5 * float(ra.abs().max())


def test_workspace_at_an_odd_address(monkeypatch):
    """Every workspace starting at byte 1 of a larger buffer: the outputs of an aligned one."""
    v, f = synthetic.icosphere(3)
    faces = T(np.asarray(f, np.int64))
    x = torch.randn((2, len(v), 3), generator=torch.Generator(device="cpu").manual_seed(3)).to(DEV)

    def run():
        S = mesh.LoopSubdivision(len(v), faces, 2)
        return [S(x), S.faces]

    want = run()
    scratch, odd = _lib.scratch, []
    monkeypatch.setattr(_lib, "scratch", lambda n, device: odd.append(n) or scratch(int(n) + 1, device)[1:])
    got = run()
    assert odd
    for a, b in zip(want, got):
        assert torch.equal(a, b)
