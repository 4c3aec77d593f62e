"""Surface sampling and face areas on the GPU (kaolin_b200.ops.mesh): parity with the reference's stored
outputs (tests/golden/sample_points.npz) through the layer below the public functions with the stored
key, full-size agreement with the numpy oracle, the public behaviour and one DMTet-style step."""
import os

import numpy as np
import pytest
import torch

from kaolin_b200 import synthetic
from kaolin_b200.metrics.trianglemesh import point_to_mesh_distance
from kaolin_b200.ops import conversions, mesh
from oracle import sample_points as osp

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sample_points.npz"))
STORED = {}
for _k in GOLDEN.files:
    _scene, _dt, _name = _k.split("/")
    _x = GOLDEN[_k]                        # index arrays are stored as int32
    STORED.setdefault((_scene, _dt), {})[_name] = _x.astype(np.int64) if _x.dtype.kind == "i" else _x
DENSE = sorted(k for k, r in STORED.items() if "first_idx" not in r)
PACKED = sorted(k for k, r in STORED.items() if "first_idx" in r)


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def key_of(k):
    return torch.tensor([int(k)], dtype=torch.int64, device=DEV)


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1.0)


# ---------------------------------------------------------------------------------------------
# Parity with the stored reference outputs.

@pytest.mark.parametrize("scene,dt", DENSE)
def test_dense_parity_with_stored_reference(scene, dt):
    r = STORED[(scene, dt)]
    v = T(r["vertices"]).requires_grad_(True)
    f = T(r["faces"])
    ff = T(r["face_features"]).requires_grad_(True) if "face_features" in r else None
    given = T(r["given_areas"]) if "given_areas" in r else None
    out = mesh._sample_points(v, f, int(r["N"]), given, ff, key_of(r["key"]))
    assert torch.equal(out[1].cpu(), T(r["choices"]).cpu())
    assert np.array_equal(out[0].detach().cpu().numpy(), r["points"])
    loss = (out[0] * T(r["grad_points"])).sum()
    if ff is not None:
        assert np.array_equal(out[2].detach().cpu().numpy(), r["features"])
        loss = loss + (out[2] * T(r["grad_features"])).sum()
    loss.backward()
    if ff is not None:
        # both sum each face's samples in ascending sample order, products rounded: bit for bit
        assert np.array_equal(ff.grad.cpu().numpy(), r["ref_grad_face_features"])
    _, u, vv = osp.uniforms(int(r["key"]), r["vertices"].shape[0], int(r["N"]), r["vertices"].dtype)
    gv, _ = osp.grad_sample_points(r["vertices"].shape, r["faces"], r["choices"], osp.weights(u, vv), r["grad_points"])
    assert rel(v.grad.cpu().numpy(), gv) <= 1e-6
    assert rel(r["ref_grad_vertices"], gv) <= 1e-6

    va = T(r["vertices"]).requires_grad_(True)
    areas = mesh.face_areas(va, f)
    assert np.array_equal(areas.detach().cpu().numpy(), r["areas"])
    areas.backward(T(r["grad_areas"]))
    got, ref = va.grad.cpu().numpy(), r["ref_grad_vertices_areas"]
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    assert rel(got[ok], osp.grad_face_areas(r["vertices"], r["faces"], r["grad_areas"])[ok]) <= 1e-5


@pytest.mark.parametrize("scene,dt", PACKED)
@pytest.mark.parametrize("counts_on_gpu", [False, True])
def test_packed_parity_with_stored_reference(scene, dt, counts_on_gpu):
    r = STORED[(scene, dt)]
    v = T(r["vertices"]).requires_grad_(True)
    first, nfm = torch.from_numpy(r["first_idx"]), torch.from_numpy(r["num_faces"])
    if counts_on_gpu:
        first, nfm = first.to(DEV), nfm.to(DEV)
    f = T(r["faces"])
    pts, ch = mesh._packed_sample_points(v, first, f, nfm, int(r["N"]), None, key_of(r["key"]))
    assert torch.equal(ch.cpu(), torch.from_numpy(r["choices"]))
    assert np.array_equal(pts.detach().cpu().numpy(), r["points"])
    (pts * T(r["grad_points"])).sum().backward()
    assert rel(v.grad.cpu().numpy(), r["ref_grad_vertices"]) <= 1e-6
    va = T(r["vertices"]).requires_grad_(True)
    areas = mesh.packed_face_areas(va, first, f, nfm)
    assert np.array_equal(areas.detach().cpu().numpy(), r["areas"])
    areas.backward(T(r["grad_areas"]))
    assert rel(va.grad.cpu().numpy(), r["ref_grad_vertices_areas"]) <= 1e-5


# ---------------------------------------------------------------------------------------------
# Full size against the oracle.

def _check_against_oracle(v_np, faces_np, N, key, dtype, out):
    """Choices equal the oracle's except where t lies within rounding of a CDF boundary; points equal
    the oracle's interpolation at the kernel's choices, bit for bit."""
    B = v_np.shape[0]
    areas = osp.face_areas(v_np, faces_np)
    r, u, vv = osp.uniforms(key, B, N, dtype)
    ch = out[1].cpu().numpy()
    F = faces_np.shape[0]
    for b in range(B):
        c = osp.cdf(areas[b])
        want, t = osp.choose(c, r[b])
        diff = np.flatnonzero(want != ch[b])
        tol = 4 * F * 2.0 ** -53 * c[-1]
        assert len(diff) <= max(2, N // 10000), len(diff)
        for i in diff:
            assert min(abs(c[want[i]] - t[i]), abs(c[ch[b, i]] - t[i])) <= tol
    w = osp.weights(u, vv)
    bi = np.arange(B)[:, None]
    pts = osp.interpolate(w, *(v_np[bi, faces_np[ch, k]] for k in range(3)))
    assert np.array_equal(out[0].cpu().numpy(), pts)


def _ico_views(level, B, dtype, seed):
    v, f = synthetic.icosphere(level)
    rng = np.random.default_rng(seed)
    v = np.stack([np.asarray(v, np.float64) * (1 + 0.3 * b) + rng.normal(scale=0.01, size=v.shape)
                  for b in range(B)]).astype(dtype)
    return v, np.asarray(f, np.int64)


@pytest.mark.parametrize("level,B,N", [(7, 1, 50000), (6, 8, 100000)])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_full_size_icospheres_against_oracle(level, B, N, dtype):
    v, f = _ico_views(level, B, dtype, level)
    key = 0x1357_9BDF_2468_ACE0
    out = mesh._sample_points(T(v), T(f), N, None, None, key_of(key))
    _check_against_oracle(v, f, N, key, dtype, out)
    assert np.array_equal(mesh.face_areas(T(v), T(f)).cpu().numpy(), osp.face_areas(v, f))


def test_view_over_2_pow_24_faces():
    n = 2897                              # 2 n^2 = 16 785 218 faces: above torch.multinomial's 2^24 limit
    g = torch.linspace(0, 1, n + 1, device=DEV, dtype=torch.float32)
    y, x = torch.meshgrid(g, g, indexing="ij")
    z = 0.05 * torch.sin(7 * x) * torch.cos(5 * y)
    verts = torch.stack([x, y, z], -1).reshape(1, -1, 3)
    i = torch.arange(n, device=DEV)
    a = (i[:, None] * (n + 1) + i[None, :]).reshape(-1)
    faces = torch.cat([torch.stack([a, a + 1, a + n + 2], 1), torch.stack([a, a + n + 2, a + n + 1], 1)])
    assert faces.shape[0] == 16785218
    N, key = 200000, 77
    out = mesh._sample_points(verts, faces, N, None, None, key_of(key))
    _check_against_oracle(verts.cpu().numpy(), faces.cpu().numpy(), N, key, np.float32, out)
    S = mesh.SurfaceSampler(verts.shape[1], faces)
    vg = verts.clone().requires_grad_(True)
    p, _ = S(vg, 1000)
    p.sum().backward()
    assert torch.isfinite(vg.grad).all() and vg.grad.abs().sum() > 0


# ---------------------------------------------------------------------------------------------
# Public behaviour.

def _sphere(dtype=torch.float32, B=2, level=3):
    v, f = _ico_views(level, B, np.float64, 3)
    return T(v).to(dtype), T(f)


def test_manual_seed_reproduces_and_reseeding_changes():
    v, f = _sphere()
    ff = torch.randn((2, f.shape[0], 3, 2), device=DEV)
    torch.manual_seed(5)
    a = mesh.sample_points(v, f, 3000, face_features=ff)
    torch.manual_seed(5)
    b = mesh.sample_points(v, f, 3000, face_features=ff)
    torch.manual_seed(6)
    c = mesh.sample_points(v, f, 3000, face_features=ff)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert not torch.equal(a[0], c[0]) and not torch.equal(a[1], c[1])


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_given_areas_equal_computed(dtype):
    v, f = _sphere(dtype)
    torch.manual_seed(1)
    a = mesh.sample_points(v, f, 2000)
    torch.manual_seed(1)
    b = mesh.sample_points(v, f, 2000, areas=mesh.face_areas(v, f))
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_gradcheck_float64():
    v, f = _sphere(torch.float64, B=2, level=1)
    areas = mesh.face_areas(v, f).detach()
    ff = torch.randn((2, f.shape[0], 3, 2), device=DEV, dtype=torch.float64, requires_grad=True)
    key = key_of(31)
    fn = lambda x, y: mesh._sample_points(x, f, 50, areas, y, key)
    assert torch.autograd.gradcheck(lambda x, y: (fn(x, y)[0], fn(x, y)[2]),
                                    (v.clone().requires_grad_(True), ff), eps=1e-6, atol=1e-8)
    assert torch.autograd.gradcheck(lambda x: mesh.face_areas(x, f), (v.clone().requires_grad_(True),), eps=1e-6,
                                    atol=1e-8)


def test_backward_is_bit_reproducible():
    v, f = _sphere(B=3, level=4)
    ff = torch.randn((3, f.shape[0], 3, 5), device=DEV)
    grads = []
    for _ in range(2):
        x, y = v.clone().requires_grad_(True), ff.clone().requires_grad_(True)
        p, _, feat = mesh._sample_points(x, f, 40000, None, y, key_of(8))
        (p.square().sum() + (feat * 1.5).sum()).backward()
        grads.append((x.grad, y.grad))
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])


def test_surface_sampler_makes_no_host_read():
    v, f = _sphere()
    S = mesh.SurfaceSampler(v.shape[1], f)
    ff = torch.randn((2, f.shape[0], 3, 3), device=DEV, requires_grad=True)
    x = v.clone().requires_grad_(True)
    torch.manual_seed(3)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        p, ch, feat = S(x, 5000, face_features=ff)
        (p.sum() + feat.sum()).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.manual_seed(3)
    q = mesh.sample_points(v, f, 5000, face_features=ff)
    assert torch.equal(p, q[0]) and torch.equal(ch, q[1]) and torch.equal(feat, q[2])
    assert torch.isfinite(x.grad).all() and torch.isfinite(ff.grad).all()


def test_surface_sampler_invalid_view_gets_nan_and_zero_gradients():
    v, f = _sphere(B=3)
    v = v.clone()
    v[1, 0, 0] = float("nan")
    x = v.requires_grad_(True)
    S = mesh.SurfaceSampler(v.shape[1], f)
    ff = torch.randn((3, f.shape[0], 3, 2), device=DEV, requires_grad=True)
    p, ch, feat = S(x, 100, face_features=ff)
    assert (ch[1] == -1).all() and torch.isnan(p[1]).all() and torch.isnan(feat[1]).all()
    assert (ch[0] >= 0).all() and torch.isfinite(p[0]).all() and torch.isfinite(p[2]).all()
    areas = mesh.face_areas(v.detach(), f)
    areas[2] = 0
    p2, ch2 = S(v.detach(), 10, areas=areas)
    assert (ch2[2] == -1).all() and (ch2[0] >= 0).all()
    (torch.nan_to_num(p).sum() + torch.nan_to_num(feat).sum()).backward()
    assert (ff.grad[1] == 0).all()


def test_errors_and_empty_cases():
    v, f = _sphere()
    with pytest.raises(ValueError):
        mesh.sample_points(v, f, 10, areas=-mesh.face_areas(v, f))
    with pytest.raises(ValueError):
        mesh.sample_points(v, f, 10, areas=torch.zeros((2, f.shape[0]), device=DEV))
    vn = v.clone()
    vn[0, 3] = float("nan")
    with pytest.raises(ValueError):
        mesh.sample_points(vn, f, 10)
    with pytest.raises(ValueError):
        mesh.sample_points(v, f, 10, areas=torch.full((2, f.shape[0]), float("inf"), device=DEV))
    bad = f.clone()
    bad[5, 1] = v.shape[1]
    with pytest.raises(IndexError):
        mesh.sample_points(v, bad, 10)
    with pytest.raises(IndexError):
        mesh.sample_points(v.clone().requires_grad_(True), bad, 10)
    with pytest.raises(IndexError):
        mesh.face_areas(v, bad)
    with pytest.raises(IndexError):
        mesh.SurfaceSampler(v.shape[1], bad)
    with pytest.raises(TypeError):
        mesh.sample_points(v.half(), f, 10)
    with pytest.raises(TypeError):
        mesh.face_areas(v.bfloat16(), f)
    with pytest.raises(TypeError):
        mesh.sample_points(v, f.int(), 10)
    with pytest.raises(TypeError):
        mesh.sample_points(v, f, 10, face_features=torch.zeros((2, f.shape[0], 3, 2), device=DEV).double())
    with pytest.raises(ValueError):
        mesh.sample_points(v, f[:0], 10)
    with pytest.raises(ValueError):
        mesh.SurfaceSampler(v.shape[1], f[:0])
    with pytest.raises(NotImplementedError):
        mesh.sample_points(v, torch.zeros((3, 4), dtype=torch.int64, device=DEV), 10)
    ff = torch.zeros((0, f.shape[0], 3, 2), device=DEV)
    p, ch, feat = mesh.sample_points(v[:0], f, 10, face_features=ff)
    assert p.shape == (0, 10, 3) and ch.shape == (0, 10) and feat.shape == (0, 10, 2)
    p, ch = mesh.sample_points(v, f, 0)
    assert p.shape == (2, 0, 3) and ch.shape == (2, 0) and ch.dtype == torch.int64
    p, ch = mesh.SurfaceSampler(v.shape[1], f)(v[:0], 7)
    assert p.shape == (0, 7, 3)
    assert mesh.face_areas(v[:0], f).shape == (0, f.shape[0])
    # an empty mesh in a packed batch is not a distribution
    with pytest.raises(ValueError):
        mesh.packed_sample_points(v[0], torch.tensor([0, 10, v.shape[1]]), f, torch.tensor([f.shape[0], 0]), 5)


def test_zero_area_gradient_is_nan_where_the_reference_is():
    r = STORED[("degenerate", "f32")]
    v = T(r["vertices"]).requires_grad_(True)
    mesh.face_areas(v, T(r["faces"])).sum().backward()
    ref = osp.grad_face_areas(r["vertices"], r["faces"], np.ones_like(r["areas"]))
    assert np.isnan(ref).any()
    assert np.array_equal(np.isnan(v.grad.cpu().numpy()), np.isnan(ref))


# ---------------------------------------------------------------------------------------------
# One DMTet-style step: marching tetrahedra -> sample_points -> point_to_mesh_distance -> backward.

def test_dmtet_step_gradient_matches_torch_chain():
    verts, tets = synthetic.freudenthal_grid(12)
    vt, tt = T(verts)[None], T(tets)
    sdf0 = (vt[0].norm(dim=-1) - 0.3).unsqueeze(0)
    tv, tf = _sphere(B=1, level=3)
    target = (tv[0] * 0.35)[tf][None]                 # (1, F, 3, 3)
    M = conversions.MarchingTetrahedra(vt.shape[1], tt)

    def step(sample):
        sdf = sdf0.clone().requires_grad_(True)
        mv, mf = M(vt, sdf)
        p = sample(mv[0][None], mf[0])
        d, _, _ = point_to_mesh_distance(p, target)
        d.mean().backward()
        return sdf.grad

    key = key_of(2718)
    keep = {}

    def ours(v, f):
        p, ch = mesh._sample_points(v, f, 20000, None, None, key)
        keep["ch"] = ch
        return p

    def chain(v, f):
        _, u, vv = osp.uniforms(2718, 1, 20000, np.float32)
        return osp.torch_points(v, f, keep["ch"], T(u), T(vv))

    g1 = step(ours)
    g2 = step(chain)
    assert torch.isfinite(g1).all() and g1.abs().sum() > 0
    assert (g1 - g2).abs().max() <= 1e-5 * max(g2.abs().max().item(), 1.0)
