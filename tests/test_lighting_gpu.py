"""sm_90a diffuse-lighting kernels against the reference's golden vectors (tests/golden/lighting.npz,
float64 outputs and gradients of kaolin.render.lighting), against an fp64 torch restatement
(oracle/lighting.py) on shaded pixels of a rendered image, and for bit-reproducible light gradients.
Tolerance 1e-5 of the tensor's scale."""
import os

import numpy as np
import pytest
import torch

from oracle import lighting as OL
from kaolin_b200 import _lib, synthetic
from kaolin_b200.render import lighting
from kaolin_b200.render.mesh import rasterize, texture_mapping

pytestmark = pytest.mark.gpu
DEV = "cuda"
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "lighting.npz"))
T = lambda k, grad=False: torch.from_numpy(np.ascontiguousarray(G[k])).float().to(DEV).requires_grad_(grad)


def close(a, ref, tol=1e-5):
    a = a.detach().double().cpu().numpy() if isinstance(a, torch.Tensor) else a
    ref = ref.detach().double().cpu().numpy() if isinstance(ref, torch.Tensor) else ref
    assert a.shape == ref.shape, (a.shape, ref.shape)
    if ref.size == 0:
        return 0.0
    scale = max(float(np.abs(ref).max()), 1e-30)
    err = float(np.abs(a - ref).max()) / scale
    assert err <= tol, err
    return err


MODELS = {"irr_ip": (lighting.sg_irradiance_inner_product, OL.sg_irradiance_inner_product, False),
          "diff_ip": (lighting.sg_diffuse_inner_product, OL.sg_diffuse_inner_product, True),
          "fitted": (lighting.sg_diffuse_fitted, OL.sg_diffuse_fitted, True)}


@pytest.mark.parametrize("L", [1, 2, 7, 8, 40])
@pytest.mark.parametrize("name", list(MODELS))
def test_sg_models_vs_reference_golden(name, L):
    fn, _, with_albedo = MODELS[name]
    keys = ("amp", "dir", "sharp", "normal") + (("albedo",) if with_albedo else ())
    ins = [T(f"L{L}_{k}", True) for k in keys]
    o = fn(*ins)
    close(o, G[f"L{L}_{name}_out"])
    (o * T(f"L{L}_w")).sum().backward()
    for k, t in zip(("g_amp", "g_dir", "g_sharp", "g_normal", "g_albedo"), ins):
        close(t.grad, G[f"L{L}_{name}_{k}"])


@pytest.mark.parametrize("nm", ["1x1", "5x3", "33x9", "70x17"])
def test_general_inner_product_vs_reference_golden(nm):
    key = f"ip{nm}"
    ins = [T(f"{key}_{k}", True) for k in ("a", "d", "s", "oa", "od", "os")]
    o = lighting.unbatched_reduced_sg_inner_product(*ins)
    close(o, G[f"{key}_out"])
    (o * T(f"{key}_w")).sum().backward()
    for k, t in zip(("a", "d", "s", "oa", "od", "os"), ins):
        close(t.grad, G[f"{key}_g_{k}"])


def test_sh9_vs_reference_golden():
    d, n, al = T("sh_direction", True), T("sh_normal", True), T("sh_albedo", True)
    o = lighting.sh9_diffuse(d, n, al)
    close(o, G["sh_diffuse_out"])
    (o * T("sh_w")).sum().backward()
    close(d.grad, G["sh_diffuse_g_direction"]); close(n.grad, G["sh_diffuse_g_normal"]); close(al.grad, G["sh_diffuse_g_albedo"])
    li, n2 = T("sh_lights", True), T("sh_normal", True)
    o = lighting.sh9_irradiance(li, n2)
    assert o.shape == (n2.shape[0],)
    close(o, G["sh_irr_out"])
    (o * T("sh_w1")).sum().backward()
    close(li.grad, G["sh_irr_g_lights"]); close(n2.grad, G["sh_irr_g_normal"])


def _image_points():
    """Normals and albedo of the covered pixels of 8 rendered icosphere views at 512^2."""
    fvz, fvi, fnz = synthetic.icosphere_views(8, 4, seed=31)
    B, F = fvz.shape[:2]
    gen = torch.Generator(device=DEV); gen.manual_seed(32)
    t = lambda a: torch.from_numpy(a).to(DEV)
    normals = torch.nn.functional.normalize(torch.randn((B, F, 3, 3), device=DEV, generator=gen), dim=-1)
    uvs = torch.rand((B, F, 3, 2), device=DEV, generator=gen)
    feat, face_idx = rasterize(512, 512, t(fvz), t(fvi), torch.cat([normals, uvs], -1))
    cov = face_idx >= 0
    tex = torch.rand((B, 3, 64, 64), device=DEV, generator=gen)
    albedo = texture_mapping(feat[..., 3:5], tex, mode="bilinear")
    n = torch.nn.functional.normalize(feat[..., :3][cov], dim=-1)
    return n.contiguous(), albedo[cov].contiguous()


def _lights(L, gen):
    amp = torch.rand((L, 3), device=DEV, generator=gen) * 2
    d = torch.nn.functional.normalize(torch.randn((L, 3), device=DEV, generator=gen), dim=-1)
    s = torch.exp(torch.rand((L,), device=DEV, generator=gen) * np.log(100.)) * 0.5
    return amp, d, s


def _run(fn, ins, w):
    ins = [t.detach().clone().requires_grad_(True) for t in ins]
    o = fn(*ins)
    (o * w).sum().backward()
    return o, [t.grad for t in ins]


@pytest.mark.parametrize("L", [1, 8, 32, 129])
def test_image_shading_vs_fp64_restatement(L):
    n, al = _image_points()
    assert n.shape[0] > 100_000
    gen = torch.Generator(device=DEV); gen.manual_seed(100 + L)
    lights = _lights(L, gen)
    w = torch.rand(n.shape, device=DEV, generator=gen) - 0.3
    for name, (fn, ref, _) in MODELS.items():
        if name == "irr_ip":
            continue
        o, grads = _run(fn, list(lights) + [n, al], w)
        ro, rgrads = _run(ref, [t.double() for t in list(lights) + [n, al]], w.double())
        close(o, ro)
        for g, rg in zip(grads[:3] + grads[4:], rgrads[:3] + rgrads[4:]):
            close(g, rg)
        keep = slice(None)
        if name == "fitted":
            # at the fitted model's two clamp kinks (mu = 1, mean = 0) fp32 and fp64 may take different sides
            kink, rounding_only = OL.fitted_kinks(*[t.double() for t in lights], n.double(), grads[4], w)
            assert rounding_only and kink.float().mean().item() < 1e-4, int(kink.sum())
            keep = ~kink
        close(grads[3][keep], rgrads[3][keep])
    o, grads = _run(lighting.sh9_diffuse, [lights[1][0], n, al], w)
    ro, rgrads = _run(OL.sh9_diffuse, [lights[1][0].double(), n.double(), al.double()], w.double())
    close(o, ro)
    for g, rg in zip(grads, rgrads):
        close(g, rg)


@pytest.mark.parametrize("model", ["diff_ip", "fitted", "sh9"])
def test_light_gradients_are_deterministic_and_independent_of_point_gradients(model):
    gen = torch.Generator(device=DEV); gen.manual_seed(7)
    N = 300_001
    n = torch.nn.functional.normalize(torch.randn((N, 3), device=DEV, generator=gen), dim=-1)
    al = torch.rand((N, 3), device=DEV, generator=gen)
    w = torch.rand((N, 3), device=DEV, generator=gen)
    if model == "sh9":
        lights, fn, w = [torch.rand((9,), device=DEV, generator=gen) - 0.5], lighting.sh9_irradiance, w[:, 0]
    else:
        lights, fn = list(_lights(8, gen)), MODELS[model][0]
    runs = []
    for point_grads in (True, True, False):
        ls = [t.clone().requires_grad_(True) for t in lights]
        pts = [n.clone().requires_grad_(point_grads)] + ([al.clone().requires_grad_(point_grads)] if model != "sh9" else [])
        (fn(*ls, *pts) * w).sum().backward()
        runs.append([t.grad for t in ls])
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)
    for a, b in zip(runs[0], runs[2]):
        assert torch.equal(a, b)


def test_general_inner_product_light_gradients_are_deterministic():
    gen = torch.Generator(device=DEV); gen.manual_seed(8)
    N, M = 100_003, 33
    ins = [torch.rand((N, 3), device=DEV, generator=gen), torch.nn.functional.normalize(torch.randn((N, 3), device=DEV, generator=gen), dim=-1),
           torch.rand((N,), device=DEV, generator=gen) * 5 + 0.5, *_lights(M, gen)]
    w = torch.rand((N, 3), device=DEV, generator=gen)
    r1 = _run(lighting.unbatched_reduced_sg_inner_product, ins, w)[1]
    r2 = _run(lighting.unbatched_reduced_sg_inner_product, ins, w)[1]
    for a, b in zip(r1[3:], r2[3:]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("N,L", [(0, 3), (5, 0), (0, 0), (1, 1), (1023, 2), (1029, 5), (4099, 1000)])
def test_edge_sizes_vs_fp64_restatement(N, L):
    gen = torch.Generator(device=DEV); gen.manual_seed(N * 7 + L)
    lights = list(_lights(L, gen))
    n = torch.nn.functional.normalize(torch.randn((N, 3), device=DEV, generator=gen), dim=-1)
    al = torch.rand((N, 3), device=DEV, generator=gen)
    w = torch.rand((N, 3), device=DEV, generator=gen)
    for name, (fn, ref, _) in MODELS.items():
        args = lights + [n] + ([al] if name != "irr_ip" else [])
        o, grads = _run(fn, args, w)
        if L == 0:          # an empty sum
            assert torch.equal(o, torch.zeros_like(o))
            assert all(g is None or torch.equal(g, torch.zeros_like(g)) for g in grads)
            continue
        ro, rgrads = _run(ref, [t.double() for t in args], w.double())
        close(o, ro)
        for g, rg in zip(grads, rgrads):
            close(g, rg)
    if L > 0:
        args = [al, n, torch.rand((N,), device=DEV, generator=gen) * 5 + 0.5] + lights
        o, grads = _run(lighting.unbatched_reduced_sg_inner_product, args, w)
        ro, rgrads = _run(OL.reduced_sg_inner_product, [t.double() for t in args], w.double())
        close(o, ro)
        for g, rg in zip(grads, rgrads):
            close(g, rg)


def test_misaligned_storage_offset():
    """Views whose base is 4 bytes past a 16-byte boundary take the scalar-load path."""
    gen = torch.Generator(device=DEV); gen.manual_seed(9)
    N, L = 2051, 3
    lights = list(_lights(L, gen))
    buf = torch.nn.functional.normalize(torch.randn((N + 1, 3), device=DEV, generator=gen), dim=-1)
    n = buf.view(-1)[1:1 + 3 * N].view(N, 3)
    assert n.data_ptr() % 16 != 0 and n.is_contiguous()
    al = torch.rand((N, 3), device=DEV, generator=gen)
    w = torch.rand((N, 3), device=DEV, generator=gen)
    for name in ("diff_ip", "fitted"):
        fn, ref, _ = MODELS[name]
        o, grads = _run(fn, lights + [n, al], w)
        o2, grads2 = _run(fn, lights + [n.clone(), al], w)      # aligned copy: the vector path
        assert torch.equal(o, o2) and all(torch.equal(a, b) for a, b in zip(grads, grads2))
        ro, rgrads = _run(ref, [t.double() for t in lights + [n, al]], w.double())
        close(o, ro)
        for g, rg in zip(grads, rgrads):
            close(g, rg)


@pytest.mark.parametrize("fn,args", [
    (lighting.sg_diffuse_inner_product, lambda: (torch.rand(2, 3), torch.rand(2, 3), torch.rand(2), torch.rand(5, 3), torch.rand(5, 3))),
    (lighting.sg_diffuse_fitted, lambda: (torch.rand(2, 3), torch.rand(2, 3), torch.rand(2), torch.rand(5, 3), torch.rand(5, 3))),
    (lighting.sg_irradiance_inner_product, lambda: (torch.rand(2, 3), torch.rand(2, 3), torch.rand(2), torch.rand(5, 3))),
    (lighting.sh9_irradiance, lambda: (torch.rand(9), torch.rand(5, 3))),
    (lighting.sh9_diffuse, lambda: (torch.rand(3), torch.rand(5, 3), torch.rand(5, 3))),
    (lighting.unbatched_reduced_sg_inner_product, lambda: (torch.rand(4, 3), torch.rand(4, 3), torch.rand(4),
                                                           torch.rand(2, 3), torch.rand(2, 3), torch.rand(2))),
])
def test_float64_inputs_are_rejected(fn, args):
    with pytest.raises(RuntimeError, match="not implemented for 'float64'"):
        fn(*[t.double().to(DEV) for t in args()])


def test_operator_shim_error_wording():
    from kaolin_b200 import _C as b200_C
    f = b200_C.render.sg.unbatched_reduced_sg_inner_product_forward_cuda
    cu = [torch.rand(4, 3, device=DEV), torch.rand(4, 3, device=DEV), torch.rand(4, device=DEV),
          torch.rand(2, 3, device=DEV), torch.rand(2, 3, device=DEV), torch.rand(2, device=DEV)]
    with pytest.raises(RuntimeError, match="expected contiguous tensor for argument direction"):
        f(cu[0], torch.rand(3, 4, device=DEV).t(), *cu[2:])
    with pytest.raises(RuntimeError, match="not implemented for 'float64'"):
        f(*[t.double() for t in cu])
    with pytest.raises(RuntimeError, match="expected tensor of size \\[4\\] for argument sharpness"):
        f(cu[0], cu[1], torch.rand(5, device=DEV), *cu[3:])
    # the public API takes non-contiguous inputs, as the reference's torch path does
    nc = torch.rand(3, 4, device=DEV).t()
    close(lighting.unbatched_reduced_sg_inner_product(cu[0], nc, *cu[2:]),
          lighting.unbatched_reduced_sg_inner_product(cu[0], nc.contiguous(), *cu[2:]), 0.0)


def test_workspace_at_an_odd_address(monkeypatch):
    """Every workspace starting at byte 1 of a larger buffer: the outputs of an aligned one."""
    gen = torch.Generator(device=DEV); gen.manual_seed(9)
    N = 10_001
    n = torch.nn.functional.normalize(torch.randn((N, 3), device=DEV, generator=gen), dim=-1)
    al = torch.rand((N, 3), device=DEV, generator=gen)
    w = torch.rand((N, 3), device=DEV, generator=gen)
    lights, sh = list(_lights(8, gen)), [torch.rand((9,), device=DEV, generator=gen) - 0.5]
    general = [al, n, torch.rand((N,), device=DEV, generator=gen) * 5 + 0.5, *_lights(5, gen)]

    def run():
        outs = []
        for fn, ins, wi in ((MODELS["diff_ip"][0], lights + [n, al], w), (MODELS["fitted"][0], lights + [n, al], w),
                            (lighting.sh9_irradiance, sh + [n], w[:, 0]),
                            (lighting.unbatched_reduced_sg_inner_product, general, w)):
            o, grads = _run(fn, ins, wi)
            outs += [o, *grads]
        return outs

    want = run()
    scratch, odd = _lib.scratch, []
    monkeypatch.setattr(_lib, "scratch", lambda n, device: odd.append(n) or scratch(int(n) + 1, device)[1:])
    got = run()
    assert odd
    for a, b in zip(want, got):
        assert torch.equal(a, b)
