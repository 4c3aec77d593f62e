"""point_to_mesh_distance on the GPU: bit-equality with the reference operator's stored outputs through
the public function and through ``_C.metrics`` driven by the reference wrapper's steps, the documented
deviations, the float64 oracle at full size, gradcheck, determinism, no host sync, workspace
alignment, peak memory and one DMTet-style loss step."""
import numpy as np
import pytest
import torch

from oracle import point_mesh_distance as oracle
from oracle import ref_golden_point_mesh as golden
from kaolin_b200 import _C, _lib, synthetic
from kaolin_b200.metrics import point_to_mesh_distance

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
SCENES = golden.scenes()
STORED = golden.load()
DT = {"f32": torch.float32, "f64": torch.float64}
CASES = [(s, dt) for s in sorted(SCENES) for dt in DT]


def _inputs(scene, dt, requires_grad=False):
    p, f, g = SCENES[scene]
    t = lambda a: torch.from_numpy(a).to(DEV, DT[dt])
    pt, ft = t(p), t(f)
    if requires_grad:
        pt.requires_grad_(True)
        ft.requires_grad_(True)
    return pt, ft, t(g)


def _public(scene, dt):
    p, f, g = _inputs(scene, dt, True)
    dist, idx, typ = point_to_mesh_distance(p, f)
    dist.backward(g)
    return {"dist": dist, "face_idx": idx, "dist_type": typ, "grad_points": p.grad, "grad_face_vertices": f.grad}


def _c_metrics(scene, dt):
    """The reference wrapper's steps (trianglemesh.py:87-99, 125-149) on ``_C.metrics``."""
    p, f, g = _inputs(scene, dt)
    out = {k: [] for k in golden.OUTPUTS}
    for b in range(p.shape[0]):
        n = p.shape[1]
        dist = torch.zeros((n,), device=DEV, dtype=p.dtype)
        idx = torch.zeros((n,), device=DEV, dtype=torch.long)
        typ = torch.zeros((n,), device=DEV, dtype=torch.int32)
        _C.metrics.unbatched_triangle_distance_forward_cuda(p[b], f[b], dist, idx, typ)
        gp, gf = torch.zeros_like(p[b]), torch.zeros_like(f[b])
        _C.metrics.unbatched_triangle_distance_backward_cuda(g[b].contiguous(), p[b], f[b], idx, typ, gp, gf)
        for k, v in zip(golden.OUTPUTS, (dist, idx, typ, gp, gf)):
            out[k].append(v)
    return {k: torch.stack(v) for k, v in out.items()}


def _bits(t):
    return t.detach().cpu().numpy().tobytes()


def _check_equal(scene, dt, ours):
    ref = STORED[(scene, dt)]
    for k in ("dist", "face_idx", "dist_type", "grad_points"):
        a = ours[k].detach().cpu().numpy()
        assert a.dtype == ref[k].dtype and a.shape == ref[k].shape, (scene, dt, k)
        assert a.tobytes() == ref[k].tobytes(), (scene, dt, k, np.argwhere(a != ref[k])[:5])
    # grad_face_vertices: bit-equal wherever a face has at most one point, else within 1e-6 of scale
    gf, rgf = ours["grad_face_vertices"].detach().cpu().numpy(), ref["grad_face_vertices"]
    idx = ref["face_idx"]
    counts = np.stack([np.bincount(idx[b], minlength=gf.shape[1]) for b in range(gf.shape[0])])
    single = counts <= 1
    assert gf[single].tobytes() == rgf[single].tobytes(), (scene, dt)
    multi = ~single
    if multi.any():
        finite = np.isfinite(rgf[multi])
        scale = max(np.abs(rgf[multi][finite]).max(initial=0.0), 1e-30)
        assert np.all(np.abs(gf[multi][finite] - rgf[multi][finite]) <= 1e-6 * scale), (scene, dt)
        np.testing.assert_array_equal(np.isfinite(gf[multi]), finite)


@pytest.mark.parametrize("scene,dt", [c for c in CASES if c[0] not in golden.DEVIATION])
@pytest.mark.parametrize("path", ["public", "c_metrics"])
def test_bit_equal_to_reference(scene, dt, path):
    _check_equal(scene, dt, (_public if path == "public" else _c_metrics)(scene, dt))


@pytest.mark.parametrize("scene,dt", [c for c in CASES if c[0] in golden.DEVIATION])
def test_nan_face_deviation(scene, dt):
    """A NaN face at a multiple of 512 does not hide the other faces: where the reference differs from
    us it returned a NaN face's result or a tile-dropped (larger) distance, and we return the smallest
    non-NaN distance; everywhere else the outputs are bit-equal."""
    ours = _public(scene, dt)
    ref = STORED[(scene, dt)]
    d, rd = ours["dist"].detach().cpu().numpy(), ref["dist"]
    i, ri = ours["face_idx"].cpu().numpy(), ref["face_idx"]
    differ = (i != ri) | (d.view(np.uint8).reshape(d.shape + (-1,)) != rd.view(np.uint8).reshape(rd.shape + (-1,))).any(-1)
    assert differ.any(), "the scene no longer shows the deviation"
    assert np.all(np.isnan(rd[differ]) | (d[differ] < rd[differ])), scene
    assert not np.isnan(d[differ]).any()
    assert np.all(ri[differ] % 512 == 0) or np.all(~np.isnan(rd[differ]))
    same = ~differ
    np.testing.assert_array_equal(ours["dist_type"].cpu().numpy()[same], ref["dist_type"][same])


def _icosphere_faces(level, rng, noise=0.0, dtype=torch.float32):
    v, f = synthetic.icosphere(level)
    v = v + noise * rng.normal(size=v.shape)
    return torch.from_numpy(v[f]).to(DEV, dtype)


def _check_oracle(p, fv, dist, idx):
    od, of, _ = oracle.point_to_mesh_distance(p.double(), fv.double())
    scale = 1.0 + (p.double() ** 2).sum(1)
    assert torch.all((dist.double() - od).abs() <= 2e-6 * scale)
    # where the faces differ, ours is a near-tie: its exact distance is within the bound of the minimum
    mine = oracle.distance_to_faces(p.double(), fv.double(), idx)
    assert torch.all((mine - od).abs() <= 2e-6 * scale)


def test_oracle_level6_icosphere_1e5_points():
    rng = np.random.default_rng(6)
    fv = _icosphere_faces(6, rng)
    d = torch.from_numpy(rng.normal(size=(100000, 3))).to(DEV)
    p = (d / d.norm(dim=1, keepdim=True) * (1 + 0.1 * torch.randn(100000, 1, device=DEV, dtype=torch.float64))).float()
    dist, idx, typ = point_to_mesh_distance(p[None], fv[None])
    sub = torch.from_numpy(rng.choice(100000, 8192, replace=False)).to(DEV)
    _check_oracle(p[sub], fv, dist[0, sub], idx[0, sub])


def test_oracle_batch_of_8_different_meshes():
    rng = np.random.default_rng(8)
    fv = torch.stack([_icosphere_faces(3, rng, noise=0.02) * (0.5 + 0.2 * b) for b in range(8)])
    p = torch.randn(8, 3000, 3, device=DEV)
    dist, idx, _ = point_to_mesh_distance(p, fv)
    for b in range(8):
        _check_oracle(p[b], fv[b], dist[b], idx[b])


def test_gradcheck_float64_away_from_region_boundaries():
    torch.manual_seed(0)
    fv = torch.tensor([[[[0., 0., 0.], [1., 0., 0.], [0., 1., 0.]], [[0., 0., 2.], [1., 0., 2.2], [0., 1., 2.1]]]],
                      device=DEV, dtype=torch.float64)
    p = torch.tensor([[[0.2, 0.2, 0.5], [-1., -1., 0.3], [2., -0.5, 0.3], [-0.5, 2., 0.3], [0.5, -1., 0.2],
                       [1., 1., 0.1], [-1., 0.5, 0.2], [0.3, 0.3, 1.8]]], device=DEV, dtype=torch.float64)
    _, _, typ = point_to_mesh_distance(p, fv)
    assert set(typ[0].tolist()) == set(range(7))
    # dist is rounded to float in float64 too (as in the reference), hence the float-sized eps and tolerances
    f = lambda a, b: point_to_mesh_distance(a, b)[0]
    assert torch.autograd.gradcheck(f, (p.requires_grad_(True), fv.requires_grad_(True)), eps=1e-3, atol=1e-3,
                                    rtol=1e-3)


def test_reruns_are_byte_identical():
    rng = np.random.default_rng(3)
    fv = _icosphere_faces(4, rng, noise=0.01).requires_grad_(True)
    p = torch.randn(2, 50000, 3, device=DEV).mul(0.3).requires_grad_(True)
    g = torch.randn(2, 50000, device=DEV)
    fv2 = fv.detach()[None].repeat(2, 1, 1, 1).requires_grad_(True)
    runs = []
    for _ in range(3):
        p.grad = fv2.grad = None
        d, i, t = point_to_mesh_distance(p, fv2)
        d.backward(g)
        runs.append([_bits(x) for x in (d, i, t, p.grad, fv2.grad)])
    assert runs[0] == runs[1] == runs[2]


def test_no_synchronising_read():
    p = torch.randn(2, 3000, 3, device=DEV, requires_grad=True)
    fv = torch.randn(2, 500, 3, 3, device=DEV, requires_grad=True)
    point_to_mesh_distance(p, fv)   # warm up (library load, allocator)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        d, _, _ = point_to_mesh_distance(p, fv)
        d.sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_workspace_at_odd_address():
    p = torch.randn(2, 700, 3, device=DEV)
    fv = torch.randn(2, 300, 3, 3, device=DEV)
    g = torch.randn(2, 700, device=DEV)
    fwd, bwd = _lib.point_mesh_distance_workspace_bytes(2, 700, 300, _lib.DTYPE_F32, "ws")
    outs = []
    for off in (0, 1):
        ws = torch.empty(max(fwd, bwd) + off, dtype=torch.uint8, device=DEV)
        d = torch.empty(2, 700, device=DEV)
        i = torch.empty(2, 700, dtype=torch.long, device=DEV)
        t = torch.empty(2, 700, dtype=torch.int32, device=DEV)
        _lib.call("dibr_b200_point_mesh_distance_forward", DEV, 2, 700, 300, _lib.DTYPE_F32, p, fv, d, i, t,
                  ws.data_ptr() + off, fwd)
        gp, gf = torch.zeros_like(p), torch.zeros_like(fv)
        _lib.call("dibr_b200_point_mesh_distance_backward", DEV, 2, 700, 300, _lib.DTYPE_F32, g, p, fv, i, t, gp, gf,
                  ws.data_ptr() + off, bwd)
        outs.append([_bits(x) for x in (d, i, t, gp, gf)])
    assert outs[0] == outs[1]


def test_peak_memory_within_layout_bound():
    rng = np.random.default_rng(5)
    fv = _icosphere_faces(5, rng)[None].repeat(2, 1, 1, 1).requires_grad_(True)
    B, N, F = 2, 2_000_000, fv.shape[1]
    assert F == 20480
    p = torch.randn(B, N, 3, device=DEV).requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    d, i, t = point_to_mesh_distance(p, fv)
    d.sum().backward()
    torch.cuda.synchronize()
    fwd, bwd = _lib.point_mesh_distance_workspace_bytes(B, N, F, _lib.DTYPE_F32, "mem")
    outputs = B * N * (4 + 8 + 4)              # dist, face_idx, dist_type
    grads = p.numel() * 4 + fv.numel() * 4 + B * N * 4   # grad_points, grad_face_vertices, grad_dist
    # both workspaces, the outputs, the gradients, and the allocator's rounding of each large block to 2 MB
    bound = fwd + bwd + outputs + grads + (16 << 20)
    assert torch.cuda.max_memory_allocated() - base <= bound


def test_empty_and_invalid():
    p = torch.randn(2, 5, 3, device=DEV)
    with pytest.raises(ValueError, match="F = 0"):
        point_to_mesh_distance(p, torch.zeros(2, 0, 3, 3, device=DEV))
    d, i, t = point_to_mesh_distance(torch.zeros(0, 5, 3, device=DEV), torch.zeros(0, 4, 3, 3, device=DEV))
    assert d.shape == i.shape == t.shape == (0, 5)
    d, i, t = point_to_mesh_distance(torch.zeros(2, 0, 3, device=DEV), torch.randn(2, 4, 3, 3, device=DEV))
    assert d.shape == (2, 0) and i.dtype == torch.long and t.dtype == torch.int32
    with pytest.raises(RuntimeError, match="not implemented for 'Half'"):
        point_to_mesh_distance(p.half(), torch.randn(2, 4, 3, 3, device=DEV).half())
    # the raw operator leaves its outputs untouched without faces, as the reference does
    dist = torch.full((5,), 7.0, device=DEV)
    idx = torch.full((5,), 3, dtype=torch.long, device=DEV)
    typ = torch.full((5,), 2, dtype=torch.int32, device=DEV)
    _C.metrics.unbatched_triangle_distance_forward_cuda(p[0], torch.zeros(0, 3, 3, device=DEV), dist, idx, typ)
    assert (dist == 7).all() and (idx == 3).all() and (typ == 2).all()


def test_non_contiguous_inputs():
    p = torch.randn(3, 400, 2, 3, device=DEV)[:, :, 0]
    fv = torch.randn(3, 3, 3, 90, device=DEV).permute(0, 3, 1, 2)
    a = point_to_mesh_distance(p, fv)
    b = point_to_mesh_distance(p.contiguous(), fv.contiguous())
    for x, y in zip(a, b):
        assert _bits(x) == _bits(y)


def test_dmtet_style_step():
    """marching_tetrahedra -> points sampled from a target icosphere -> point_to_mesh_distance().mean() ->
    backward to the SDF; against the same step with the distance in float64.  The float32 face gradients
    of small faces carry the cancellation of the normal's normalisation; the measured difference is
    about 2e-5 of the gradient's scale on an H100, so the bound is 1e-4."""
    from kaolin_b200.ops.conversions import marching_tetrahedra
    res = 12
    grid_v, tets = synthetic.freudenthal_grid(res)
    verts = torch.from_numpy(np.asarray(grid_v, np.float32)).to(DEV)[None] * 2
    tets = torch.from_numpy(np.asarray(tets, np.int64)).to(DEV)
    rng = np.random.default_rng(11)
    sdf0 = (verts[0].norm(dim=1) - 0.6 + 0.01 * torch.from_numpy(rng.normal(size=verts.shape[1])).to(DEV).float())
    tv, tf = synthetic.icosphere(3)
    target = torch.from_numpy((tv * 0.7)[tf].mean(1)).to(DEV)          # face centres of a target sphere

    def step(dtype):
        sdf = sdf0[None].clone().requires_grad_(True)
        mv, mf = marching_tetrahedra(verts, tets, sdf)
        fv = mv[0][mf[0]].to(dtype)
        d, _, _ = point_to_mesh_distance(target.to(dtype)[None], fv[None])
        d.mean().backward()
        return sdf.grad

    g32, g64 = step(torch.float32), step(torch.float64)
    assert torch.isfinite(g32).all() and g32.abs().max() > 0
    assert (g32 - g64).abs().max() <= 1e-4 * g64.abs().max()
