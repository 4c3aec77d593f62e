"""TEST INFRASTRUCTURE — the diffuse-lighting formulas of kaolin/render/lighting/sg.py and sh.py,
restated in torch from the mathematics (dtype of the inputs: float64 for the tests' reference,
float32 for the benchmark's "reference formulation" row).  Autograd through these gives the
reference gradients.  Never imported by kaolin_b200."""
import math

import torch


def sg_pairs(a, d, s, oa, od, os_):
    """<sg_n, other_m> for every pair: (N, M, 3)."""
    v = s[:, None, None] * d[:, None, :] + os_[None, :, None] * od[None, :, :]
    um = torch.sqrt((v * v).sum(-1, keepdim=True))
    lm = (s[:, None] + os_[None, :])[..., None]
    return 2 * math.pi * torch.exp(um - lm) * (a[:, None, :] * oa[None, :, :]) * (1 - torch.exp(-2 * um)) / um


def reduced_sg_inner_product(a, d, s, oa, od, os_):
    return sg_pairs(a, d, s, oa, od, os_).sum(1)


def sg_irradiance_inner_product(amp, dirs, sharp, normal):
    lobe_a = torch.full_like(normal, 1.17)
    lobe_s = torch.full_like(normal[:, 0], 2.133)
    return torch.clamp(reduced_sg_inner_product(lobe_a, normal, lobe_s, amp, dirs, sharp), min=0.)


def sg_diffuse_inner_product(amp, dirs, sharp, normal, albedo):
    return sg_irradiance_inner_product(amp, dirs, sharp, normal) * (albedo / math.pi)


def sg_irradiance_fitted(amp, dirs, sharp, normal, magnitude=False):
    """Stephen Hill's fitted SG irradiance per (point, light): (N, L, 3).  With ``magnitude``, the
    magnitude of its parts instead, (|scale y| + |bias|) |2 pi amp / sharp|: the scale of its rounding."""
    mu = normal @ dirs.t()
    lb = sharp[None, :]
    eml = torch.exp(-lb)
    em2l = eml * eml
    rl = 1. / lb
    scale = 1. + 2. * em2l - rl
    bias = (eml - em2l) * rl - em2l
    x = torch.sqrt(1. - scale)
    x0 = 0.36 * mu
    x1 = x / (4. * 0.36)
    n = x0 + x1
    y = torch.where(torch.abs(x0) <= x1, n * n / x, torch.clamp(mu, min=0., max=1.))
    if magnitude:
        return ((scale * y).abs() + bias.abs())[..., None] * (2 * math.pi * amp / sharp[:, None]).abs()[None]
    return (scale * y + bias)[..., None] * (2 * math.pi * amp / sharp[:, None])[None]


def fitted_kinks(amp, dirs, sharp, normal, grad_albedo, grad_out):
    """Points where an fp32 sg_diffuse_fitted may take the other side of a gradient kink than fp64:

    * clamp(mu, 0, 1) at mu = 1: a normal pointing at a light gives n . d within rounding of 1, and
      torch's clamp passes the gradient at the bound but not above it;
    * clamp(mean, min=0): the fitted irradiance can be negative.  The fp32 side is read off
      ``grad_albedo`` (grad_out * clamp(mean) / pi is 0 exactly where the clamp cut, if grad_out != 0).

    Returns (points, whether every clamp(min=0) flip has its fp64 mean within fp32 rounding of 0:
    (L + 16) 2^-23 times the mean magnitude of the summed parts)."""
    at_one = ((normal @ dirs.t() - 1).abs() <= 1e-6).any(1)
    mean = sg_irradiance_fitted(amp, dirs, sharp, normal).mean(1)
    mag = sg_irradiance_fitted(amp, dirs, sharp, normal, magnitude=True).mean(1)
    flip = (grad_out != 0) & ((grad_albedo != 0) != (mean > 0))
    bound = (amp.shape[0] + 16) * 2.0 ** -23 * mag
    return at_one | flip.any(1), bool((mean.abs()[flip] <= bound[flip]).all())


def sg_diffuse_fitted(amp, dirs, sharp, normal, albedo):
    return torch.clamp(sg_irradiance_fitted(amp, dirs, sharp, normal).mean(1), min=0.) * (albedo / math.pi)


def project_onto_sh9(d):
    x, y, z = d[..., 0], d[..., 1], d[..., 2]
    c1 = math.sqrt(3 / (4 * math.pi))
    c2 = math.sqrt(15 / (4 * math.pi))
    return torch.stack([torch.full_like(x, 0.5 / math.sqrt(math.pi)), -c1 * y, c1 * z, -c1 * x,
                        c2 * x * y, -c2 * y * z, math.sqrt(5 / (16 * math.pi)) * (3 * z * z - 1),
                        -c2 * x * z, math.sqrt(15 / (16 * math.pi)) * (x * x - y * y)], -1)


_SH9_BAND = [math.pi] + [2 * math.pi / 3] * 3 + [math.pi / 4] * 5


def sh9_irradiance(lights, normals):
    b = project_onto_sh9(normals) * torch.tensor(_SH9_BAND, dtype=normals.dtype, device=normals.device)
    return (b * lights[None, :]).sum(-1)


def sh9_diffuse(directions, normals, albedo):
    return albedo * sh9_irradiance(project_onto_sh9(directions), normals)[:, None]
