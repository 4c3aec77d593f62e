"""Regenerates tests/golden/specular.npz from the reference (run where its sources are present).

    python tests/golden/make_specular_golden.py

Outputs and autograd gradients of the reference's OWN functions, imported in place, in float64 on
seeded inputs: kaolin.render.lighting.sg sg_warp_specular_term (sg.py:293-350) with the gradients
of all seven inputs, and its building blocks sg_distribution_term, sg_warp_distribution and fresnel
(sg.py:220-291).  Under the stub ``_C`` the reference's fused inner-product operator returns None for
8 or more lights, so for those sizes the module's ``unbatched_reduced_sg_inner_product`` is rebound
to the reference's own composition that the operator fuses, ``unbatched_sg_inner_product(...).sum(1)``
(sg.py:676-679); ``sg_warp_specular_term`` itself then runs unchanged.

Points: unit view directions; normals with n.v in [0.25, 1] (unit, or of norm 0.8-1.2), and unit
normals facing away from the view (n.v in [-1, -0.2]: zero output); roughness in [0.3, 1].
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))
from oracle import ref_import  # noqa: E402

sg = ref_import.module("kaolin.render.lighting.sg")
_fused = sg.unbatched_reduced_sg_inner_product
D = torch.float64
g = torch.Generator().manual_seed(20261016)


def unit(n):
    v = torch.randn((n, 3), generator=g, dtype=D)
    return v / v.norm(dim=1, keepdim=True)


def lights(L):
    amp = torch.rand((L, 3), generator=g, dtype=D) * 3
    dirs = unit(L)
    sharp = torch.exp(torch.rand((L,), generator=g, dtype=D) * np.log(100.)) * 0.5   # 0.5 .. 50
    return amp, dirs, sharp


def points(N):
    view = unit(N)
    t = unit(N)
    t = t - (t * view).sum(1, keepdim=True) * view
    t = t / t.norm(dim=1, keepdim=True)
    cos = 0.25 + 0.75 * torch.rand((N, 1), generator=g, dtype=D)
    cos[:8] = -(0.2 + 0.8 * torch.rand((8, 1), generator=g, dtype=D))                 # facing away
    normal = cos * view + torch.sqrt(1 - cos * cos) * t
    normal[16:48] *= 0.8 + 0.4 * torch.rand((32, 1), generator=g, dtype=D)            # non-unit normals
    roughness = 0.3 + 0.7 * torch.rand((N,), generator=g, dtype=D)
    spec_albedo = torch.rand((N, 3), generator=g, dtype=D)
    return normal, roughness, view, spec_albedo


out = {}
N = 96
for L in (1, 2, 7, 8, 40):
    sg.unbatched_reduced_sg_inner_product = _fused if L < 8 else (
        lambda *a: sg.unbatched_sg_inner_product(*a).sum(1))
    ins = lights(L) + points(N)
    w = torch.rand((N, 3), generator=g, dtype=D) - 0.3
    for k, t in zip(("amp", "dir", "sharp", "normal", "roughness", "view", "spec_albedo"), ins):
        out[f"L{L}_{k}"] = t
    out[f"L{L}_w"] = w
    leaves = [t.clone().requires_grad_(True) for t in ins]
    o = sg.sg_warp_specular_term(*leaves)
    (o * w).sum().backward()
    out[f"L{L}_out"] = o.detach()
    for k, t in zip(("amp", "dir", "sharp", "normal", "roughness", "view", "spec_albedo"), leaves):
        out[f"L{L}_g_{k}"] = t.grad
    assert (o[:8] == 0).all() and (o[8:] > 0).any(), L
sg.unbatched_reduced_sg_inner_product = _fused

normal, roughness, view, spec_albedo = points(N)
amp, dirs, sharp = sg.sg_distribution_term(normal, roughness)
wa, wd, ws = sg.sg_warp_distribution(amp, dirs, sharp, view)
ldh = torch.rand((N, 1), generator=g, dtype=D)
out.update(bb_normal=normal, bb_roughness=roughness, bb_view=view, bb_spec_albedo=spec_albedo, bb_ldh=ldh,
           bb_ndf_amp=amp, bb_ndf_dir=dirs, bb_ndf_sharp=sharp, bb_warp_amp=wa, bb_warp_dir=wd, bb_warp_sharp=ws,
           bb_fresnel=sg.fresnel(ldh, spec_albedo))

out = {k: v.detach().contiguous().numpy() for k, v in out.items()}
np.savez_compressed(os.path.join(HERE, "specular.npz"), **out)
print("wrote", os.path.join(HERE, "specular.npz"), len(out), "arrays")
