"""Regenerates tests/golden/lighting.npz from the reference (run in the build container only).

    python tests/golden/make_lighting_golden.py

Outputs and autograd gradients of the reference's OWN functions, imported in place, in float64 on
seeded inputs:
  kaolin.render.lighting.sg  sg_irradiance_inner_product, sg_diffuse_inner_product,
                             sg_diffuse_fitted, unbatched_reduced_sg_inner_product   sg.py:389-680
  kaolin.render.lighting.sh  project_onto_sh9, sh9_irradiance, sh9_diffuse          sh.py:28-123
Under the stub ``_C`` the reference's fused operator returns None for 8 or more "other" lobes, so for
those sizes the golden is the reference's own composition that the operator fuses:
``unbatched_sg_inner_product(...).sum(1)`` (sg.py:676-679), then clamp and albedo / pi (sg.py:514-558).
"""
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))
from oracle import ref_import  # noqa: E402

sg = ref_import.module("kaolin.render.lighting.sg")
sh = ref_import.module("kaolin.render.lighting.sh")
D = torch.float64
g = torch.Generator().manual_seed(20261015)


def reduced(a, d, s, oa, od, os_):
    if oa.shape[0] < 8:
        return sg.unbatched_reduced_sg_inner_product(a, d, s, oa, od, os_)
    return sg.unbatched_sg_inner_product(a, d, s, oa, od, os_).sum(1)


def irradiance_ip(amp, dirs, sharp, normal):
    if amp.shape[0] < 8:
        return sg.sg_irradiance_inner_product(amp, dirs, sharp, normal)
    la, ld, ls = sg.cosine_lobe_sg(normal)
    return torch.clamp(reduced(la, ld, ls, amp, dirs, sharp), min=0.)


def diffuse_ip(amp, dirs, sharp, normal, albedo):
    if amp.shape[0] < 8:
        return sg.sg_diffuse_inner_product(amp, dirs, sharp, normal, albedo)
    return irradiance_ip(amp, dirs, sharp, normal) * (albedo / math.pi)


def unit(n):
    v = torch.randn((n, 3), generator=g, dtype=D)
    return v / v.norm(dim=1, keepdim=True)


def lights(L):
    amp = torch.rand((L, 3), generator=g, dtype=D) * 3
    dirs = unit(L)
    sharp = torch.exp(torch.rand((L,), generator=g, dtype=D) * math.log(100.)) * 0.5   # 0.5 .. 50
    return amp, dirs, sharp


out = {}
N = 96
for L in (1, 2, 7, 8, 40):
    amp, dirs, sharp = lights(L)
    normal = unit(N) * (0.6 + 0.8 * torch.rand((N, 1), generator=g, dtype=D))      # non-unit normals
    normal[:8] = -dirs[0] * (0.5 + torch.rand((8, 1), generator=g, dtype=D))       # facing away from light 0
    normal[8:12] = -dirs.mean(0) / dirs.mean(0).norm()                              # away from all of them
    albedo = torch.rand((N, 3), generator=g, dtype=D)
    w = torch.rand((N, 3), generator=g, dtype=D) - 0.3
    out.update({f"L{L}_amp": amp, f"L{L}_dir": dirs, f"L{L}_sharp": sharp, f"L{L}_normal": normal,
                f"L{L}_albedo": albedo, f"L{L}_w": w})
    for name, fn, with_albedo in (("irr_ip", irradiance_ip, False), ("diff_ip", diffuse_ip, True),
                                  ("fitted", sg.sg_diffuse_fitted, True)):
        ins = [t.clone().requires_grad_(True) for t in (amp, dirs, sharp, normal) + ((albedo,) if with_albedo else ())]
        o = fn(*ins)
        (o * w).sum().backward()
        out[f"L{L}_{name}_out"] = o.detach()
        for k, t in zip(("g_amp", "g_dir", "g_sharp", "g_normal", "g_albedo"), ins):
            out[f"L{L}_{name}_{k}"] = t.grad
    if L in (2, 8):
        # fitted branches: |x0| <= x1 holds for some pairs and not for others
        lb = sharp[None]
        eml = torch.exp(-lb); em2l = eml * eml
        x = torch.sqrt(1. - (1. + 2. * em2l - 1. / lb))
        br = (0.36 * (normal @ dirs.t())).abs() <= x / 1.44
        assert br.any() and (~br).any(), L

for (n, m) in ((1, 1), (5, 3), (33, 9), (70, 17)):
    ins = [torch.rand((n, 3), generator=g, dtype=D) * 2, unit(n), torch.rand((n,), generator=g, dtype=D) * 10 + 0.5,
           torch.rand((m, 3), generator=g, dtype=D) * 2, unit(m), torch.rand((m,), generator=g, dtype=D) * 10 + 0.5]
    ins = [t.requires_grad_(True) for t in ins]
    w = torch.rand((n, 3), generator=g, dtype=D) - 0.3
    o = reduced(*ins)
    (o * w).sum().backward()
    key = f"ip{n}x{m}"
    for k, t in zip(("a", "d", "s", "oa", "od", "os"), ins):
        out[f"{key}_{k}"] = t.detach()
        out[f"{key}_g_{k}"] = t.grad
    out[f"{key}_w"] = w
    out[f"{key}_out"] = o.detach()

direction = torch.tensor([0.3, -0.5, 0.8], dtype=D)
direction = (direction / direction.norm()).requires_grad_(True)
normal = (unit(N) * (0.6 + 0.8 * torch.rand((N, 1), generator=g, dtype=D))).requires_grad_(True)
albedo = torch.rand((N, 3), generator=g, dtype=D).requires_grad_(True)
w = torch.rand((N, 3), generator=g, dtype=D) - 0.3
o = sh.sh9_diffuse(direction, normal, albedo)
(o * w).sum().backward()
out.update(sh_direction=direction.detach(), sh_normal=normal.detach(), sh_albedo=albedo.detach(), sh_w=w,
           sh_diffuse_out=o.detach(), sh_diffuse_g_direction=direction.grad, sh_diffuse_g_normal=normal.grad,
           sh_diffuse_g_albedo=albedo.grad)
lights9 = (torch.rand((9,), generator=g, dtype=D) - 0.5).requires_grad_(True)
n2 = normal.detach().clone().requires_grad_(True)
w1 = torch.rand((N,), generator=g, dtype=D) - 0.3
o = sh.sh9_irradiance(lights9, n2)
(o * w1).sum().backward()
out.update(sh_lights=lights9.detach(), sh_w1=w1, sh_irr_out=o.detach(), sh_irr_g_lights=lights9.grad,
           sh_irr_g_normal=n2.grad, sh_project=sh.project_onto_sh9(direction.detach()))

out = {k: v.detach().numpy() for k, v in out.items()}
np.savez_compressed(os.path.join(HERE, "lighting.npz"), **out)
print("wrote", os.path.join(HERE, "lighting.npz"), len(out), "arrays")
