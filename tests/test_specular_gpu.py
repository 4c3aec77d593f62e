"""sg_warp_specular_term on its sm_90a kernels: against the reference's golden vectors
(tests/golden/specular.npz, float64 outputs and gradients of kaolin.render.lighting), against the
fp64 restatement (oracle/specular.py) on shaded pixels of rendered, textured views, against the
reference's structure composed from this library's SG inner product, and for bit-reproducible light
gradients.  Tolerance 1e-5 of the tensor's scale where the formula is well conditioned in fp32."""
import os

import numpy as np
import pytest
import torch

from oracle import specular as OS
from kaolin_b200 import _lib, synthetic
from kaolin_b200.render import lighting
from kaolin_b200.render.mesh import rasterize, texture_mapping

pytestmark = pytest.mark.gpu
DEV = "cuda"
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "specular.npz"))
T = lambda k, grad=False: torch.from_numpy(np.ascontiguousarray(G[k])).float().to(DEV).requires_grad_(grad)
INPUTS = ("amp", "dir", "sharp", "normal", "roughness", "view", "spec_albedo")


def err(a, ref):
    a, ref = a.detach().double().cpu(), ref.detach().double().cpu()
    assert a.shape == ref.shape, (a.shape, ref.shape)
    if ref.numel() == 0:
        return 0.0
    return float((a - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)


def close(a, ref, tol=1e-5):
    e = err(a, ref)
    assert e <= tol, e
    return e


def _run(fn, ins, w):
    ins = [t.detach().clone().requires_grad_(True) for t in ins]
    o = fn(*ins)
    (o * w).sum().backward()
    return o, [t.grad for t in ins]


def _lights(L, gen):
    amp = torch.rand((L, 3), device=DEV, generator=gen) * 2
    d = torch.nn.functional.normalize(torch.randn((L, 3), device=DEV, generator=gen), dim=-1)
    s = torch.exp(torch.rand((L,), device=DEV, generator=gen) * np.log(100.)) * 0.5
    return [amp, d, s]


def _points(N, gen):
    """Well-conditioned points: unit view, unit normal with n.v in [0.2, 1], roughness in [0.3, 1]."""
    v = torch.nn.functional.normalize(torch.randn((N, 3), device=DEV, generator=gen), dim=-1)
    t = torch.randn((N, 3), device=DEV, generator=gen)
    t = torch.nn.functional.normalize(t - (t * v).sum(1, keepdim=True) * v, dim=-1)
    c = 0.2 + 0.8 * torch.rand((N, 1), device=DEV, generator=gen)
    n = c * v + torch.sqrt(1 - c * c) * t
    r = 0.3 + 0.7 * torch.rand((N,), device=DEV, generator=gen)
    return [n, r, v, torch.rand((N, 3), device=DEV, generator=gen)]


@pytest.mark.parametrize("L", [1, 2, 7, 8, 40])
def test_specular_vs_reference_golden(L):
    ins = [T(f"L{L}_{k}", True) for k in INPUTS]
    o = lighting.sg_warp_specular_term(*ins)
    close(o, torch.from_numpy(G[f"L{L}_out"]))
    (o * T(f"L{L}_w")).sum().backward()
    for k, t in zip(INPUTS, ins):
        close(t.grad, torch.from_numpy(G[f"L{L}_g_{k}"]))


def _image_points():
    """Normal, roughness, view and spec albedo of the covered pixels of 8 rendered icosphere views at
    512^2: roughness (0.02 .. 1) and spec albedo through texture_mapping, the view from per-pixel
    pinhole rays."""
    fvz, fvi, fnz = synthetic.icosphere_views(8, 4, seed=41)
    B, F = fvz.shape[:2]
    H = W = 512
    gen = torch.Generator(device=DEV); gen.manual_seed(42)
    t = lambda a: torch.from_numpy(a).to(DEV)
    normals = torch.nn.functional.normalize(torch.randn((B, F, 3, 3), device=DEV, generator=gen), dim=-1)
    uvs = torch.rand((B, F, 3, 2), device=DEV, generator=gen)
    feat, face_idx = rasterize(H, W, t(fvz), t(fvi), torch.cat([normals, uvs], -1))
    cov = face_idx >= 0
    rough = texture_mapping(feat[..., 3:5], 0.02 + 0.98 * torch.rand((B, 1, 64, 64), device=DEV, generator=gen),
                            mode="bilinear")
    spec = texture_mapping(feat[..., 3:5], torch.rand((B, 3, 64, 64), device=DEV, generator=gen), mode="bilinear")
    ys, xs = torch.meshgrid(torch.arange(H, device=DEV), torch.arange(W, device=DEV), indexing="ij")
    tan = 0.6
    rays = torch.stack([((xs + 0.5) / W * 2 - 1) * tan, -((ys + 0.5) / H * 2 - 1) * tan, -torch.ones_like(xs, dtype=torch.float32)], -1)
    view = -torch.nn.functional.normalize(rays, dim=-1)[None].expand(B, -1, -1, -1)
    n = torch.nn.functional.normalize(feat[..., :3][cov], dim=-1)
    return [n.contiguous(), rough[cov][:, 0].contiguous(), view[cov].contiguous(), spec[cov].contiguous()]


def _kinks(n, r, v):
    """Points whose fp64 n.v, n.w or ldh lie within 1e-5 of a clamp bound, where fp32 may take the
    other side of the clamp and its gradient jumps."""
    n, r, v = n.double(), r.double(), v.double()
    nv = (n * v).sum(1)
    w = -v + 2 * nv[:, None] * n
    ndl = (n * w).sum(1)
    h = torch.nn.functional.normalize(w + v, dim=-1)
    ldh = (w * h).sum(1)
    near = lambda x, b: (x - b).abs() <= 1e-5
    return near(nv, 0) | near(nv, 1e-4) | near(nv, 1) | near(ndl, 0) | near(ndl, 1) | near(ldh, 0) | near(ldh, 1)


@pytest.mark.parametrize("L", [1, 8, 32, 129])
def test_image_shading_vs_fp64_restatement(L):
    pts = _image_points()
    n, r, v, s = pts
    assert n.shape[0] > 100_000
    gen = torch.Generator(device=DEV); gen.manual_seed(200 + L)
    lights = _lights(L, gen)
    w = torch.rand(n.shape, device=DEV, generator=gen) - 0.3
    good = (r >= 0.3) & ((n * v).sum(1) >= 0.2)
    assert 0.2 < good.float().mean().item() < 0.8
    # well-conditioned tier: every output and gradient within 1e-5 of scale.  The roughness gradient
    # is -(g_a a + g_ws ws) / m2 plus the Smith terms, and the lobe's amplitude and sharpness terms
    # nearly cancel: there it is held to 1e-5 or to 4x the reference formula evaluated in fp32.
    sub = lights + [t[good] for t in pts]
    o, grads = _run(lighting.sg_warp_specular_term, sub, w[good])
    ro, rgrads = _run(OS.sg_warp_specular_term, [t.double() for t in sub], w[good].double())
    close(o, ro)
    for i, (g, rg) in enumerate(zip(grads, rgrads)):
        if i != 4:
            close(g, rg)
    r32 = _run(OS.sg_warp_specular_term, sub, w[good])[1][4]
    assert err(grads[4], rgrads[4]) <= max(1e-5, 4 * err(r32, rgrads[4])), (err(grads[4], rgrads[4]), err(r32, rgrads[4]))
    # all points: no worse than 4x the reference formula evaluated in fp32, plus 1e-5 of scale
    ins = lights + pts
    o, grads = _run(lighting.sg_warp_specular_term, ins, w)
    o32, grads32 = _run(OS.sg_warp_specular_term, ins, w)
    ro, rgrads = _run(OS.sg_warp_specular_term, [t.double() for t in ins], w.double())
    kink = _kinks(n, r, v)
    assert kink.float().mean().item() < 1e-3, int(kink.sum())
    for i, (a, b, ref) in enumerate(zip([o] + grads, [o32] + grads32, [ro] + rgrads)):
        if i >= 4:          # per-point gradients: away from the clamp kinks
            a, b, ref = a[~kink], b[~kink], ref[~kink]
        assert err(a, ref) <= 4 * err(b, ref) + 1e-5, (i, err(a, ref), err(b, ref))


def test_fused_kernel_matches_the_composed_reference_structure():
    """The torch prologue, this library's unbatched_reduced_sg_inner_product and the torch epilogue."""
    gen = torch.Generator(device=DEV); gen.manual_seed(11)
    ins = _lights(24, gen) + _points(50_001, gen)
    w = torch.rand((50_001, 3), device=DEV, generator=gen)
    o, grads = _run(lighting.sg_warp_specular_term, ins, w)
    composed = lambda *a: OS.sg_warp_specular_term(*a, inner=lighting.unbatched_reduced_sg_inner_product)
    co, cgrads = _run(composed, ins, w)
    close(o, co)
    for g, cg in zip(grads, cgrads):
        close(g, cg)


def test_light_gradients_are_deterministic_and_independent_of_point_gradients():
    gen = torch.Generator(device=DEV); gen.manual_seed(12)
    N = 300_001
    lights, pts = _lights(8, gen), _points(N, gen)
    w = torch.rand((N, 3), device=DEV, generator=gen)
    runs = []
    for point_grads in (True, True, False):
        ls = [t.clone().requires_grad_(True) for t in lights]
        ps = [t.clone().requires_grad_(point_grads) for t in pts]
        (lighting.sg_warp_specular_term(*ls, *ps) * w).sum().backward()
        runs.append([t.grad for t in ls])
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)
    for a, b in zip(runs[0], runs[2]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("N,L", [(0, 3), (5, 0), (0, 0), (1, 1), (1023, 2), (1029, 5), (4099, 1000)])
def test_edge_sizes_vs_fp64_restatement(N, L):
    gen = torch.Generator(device=DEV); gen.manual_seed(N * 7 + L)
    ins = _lights(L, gen) + _points(N, gen)
    w = torch.rand((N, 3), device=DEV, generator=gen)
    o, grads = _run(lighting.sg_warp_specular_term, ins, w)
    if L == 0:          # an empty sum
        assert torch.equal(o, torch.zeros_like(o))
        assert all(torch.equal(g, torch.zeros_like(g)) for g in grads)
        return
    ro, rgrads = _run(OS.sg_warp_specular_term, [t.double() for t in ins], w.double())
    close(o, ro)
    for g, rg in zip(grads, rgrads):
        close(g, rg)


def test_misaligned_and_non_contiguous_inputs():
    """Views whose base is 4 bytes past a 16-byte boundary take the scalar-load path and give the bits
    of an aligned copy; non-contiguous inputs are accepted."""
    gen = torch.Generator(device=DEV); gen.manual_seed(13)
    N = 2051
    lights = _lights(3, gen)
    n, r, v, s = _points(N, gen)
    buf = torch.empty((N + 1) * 3, device=DEV)
    nm = buf[1:1 + 3 * N].view(N, 3)
    nm.copy_(n)
    assert nm.data_ptr() % 16 != 0 and nm.is_contiguous()
    w = torch.rand((N, 3), device=DEV, generator=gen)
    o, grads = _run(lighting.sg_warp_specular_term, lights + [nm, r, v, s], w)
    o2, grads2 = _run(lighting.sg_warp_specular_term, lights + [n, r, v, s], w)
    assert torch.equal(o, o2) and all(torch.equal(a, b) for a, b in zip(grads, grads2))
    vt = v.t().contiguous().t()
    assert not vt.is_contiguous()
    assert torch.equal(lighting.sg_warp_specular_term(*lights, n, r, vt, s), o2)


def test_float64_inputs_are_rejected():
    gen = torch.Generator(device=DEV); gen.manual_seed(14)
    ins = _lights(2, gen) + _points(5, gen)
    with pytest.raises(RuntimeError, match="not implemented for 'float64'"):
        lighting.sg_warp_specular_term(*[t.double() for t in ins])


def test_workspace_at_an_odd_address(monkeypatch):
    """Every workspace starting at byte 1 of a larger buffer: the outputs of an aligned one."""
    gen = torch.Generator(device=DEV); gen.manual_seed(9)
    N = 10_001
    ins, w = _lights(8, gen) + _points(N, gen), torch.rand((N, 3), device=DEV, generator=gen)

    def run():
        o, grads = _run(lighting.sg_warp_specular_term, ins, w)
        return [o, *grads]

    want = run()
    scratch, odd = _lib.scratch, []
    monkeypatch.setattr(_lib, "scratch", lambda n, device: odd.append(n) or scratch(int(n) + 1, device)[1:])
    got = run()
    assert odd
    for a, b in zip(want, got):
        assert torch.equal(a, b)
