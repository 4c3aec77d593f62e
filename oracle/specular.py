"""TEST INFRASTRUCTURE — the specular term of kaolin/render/lighting/sg.py (sg_warp_specular_term),
restated in torch from the mathematics: float64 inputs for the tests' reference, float32 for the
benchmark's "reference formulation" row.  Autograd through it gives the reference gradients.
Never imported by kaolin_b200.

The term is split where the reference's own structure splits it: the per-point lobe (``lobe``), the
sum of its SG inner products with the lights (``inner``, by default the restatement in
oracle/lighting.py), and the per-point epilogue (``epilogue``)."""
import math

import torch

from . import lighting as OL


def _dot(a, b):
    return (a * b).sum(-1, keepdim=True)


def lobe(normal, roughness, view):
    """The GGX distribution lobe of (normal, roughness) warped by the view: amplitude (N, 3),
    direction w (N, 3), sharpness (N,)."""
    m2 = roughness * roughness
    amp = (1. / (math.pi * m2))[:, None].expand(-1, 3)
    w = -view - 2 * _dot(-view, normal) * normal
    sharp = (2. / m2) / (4. * torch.clamp(_dot(normal, view)[:, 0], min=1e-4))
    return amp, w, sharp


def _smith(m2, x):
    return 1. / (x + torch.sqrt(m2 + (1. - m2) * x * x))


def epilogue(acc, normal, roughness, view, w, spec_albedo):
    ndl = torch.clamp(_dot(normal, w), min=0., max=1.)
    ndv = torch.clamp(_dot(normal, view), min=0., max=1.)
    h = w + view
    ldh = torch.clamp(_dot(w, h / torch.sqrt(_dot(h, h))), min=0., max=1.)
    m2 = (roughness * roughness)[:, None]
    out = acc * (_smith(m2, ndl) * _smith(m2, ndv))
    out = out * (spec_albedo + (1. - spec_albedo) * torch.pow(1. - ldh, 5))
    return torch.clamp(out * ndl, min=0.)


def sg_warp_specular_term(amp, dirs, sharp, normal, roughness, view, spec_albedo,
                          inner=OL.reduced_sg_inner_product):
    la, lw, ls = lobe(normal, roughness, view)
    return epilogue(inner(la, lw, ls, amp, dirs, sharp), normal, roughness, view, lw, spec_albedo)
