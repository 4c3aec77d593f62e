"""Spherical-Gaussian lighting — drop-ins for kaolin.render.lighting.sg
(``unbatched_reduced_sg_inner_product``, ``sg_irradiance_inner_product``,
``sg_diffuse_inner_product``, ``sg_diffuse_fitted``, ``sg_warp_specular_term``).  Each is one sm_90a
kernel each way (kaolin_b200/csrc/lighting.cu) instead of the reference's chains of torch kernels and
their (N, L, 3) temporaries.  Same signatures, shape assertions and return shapes.  The building
blocks of the specular term (``sg_distribution_term``, ``sg_warp_distribution``, ``fresnel``) are
plain torch and run on any device.

Inputs must be float32 CUDA tensors.  The reference's operator is float-only too, but below 8 lights
its torch path would also accept float64; here float64 raises RuntimeError.
"""
import math

import torch
from torch.autograd import Function

from ... import _lib
from ..mesh import _host

__all__ = ["unbatched_reduced_sg_inner_product", "sg_irradiance_inner_product", "sg_diffuse_inner_product",
           "sg_diffuse_fitted", "sg_distribution_term", "sg_warp_distribution", "fresnel", "sg_warp_specular_term"]


def _c(t):
    return None if t is None else t.contiguous()


class UnbatchedReducedSgInnerProductB200(Function):
    @staticmethod
    def forward(ctx, amplitude, direction, sharpness, other_amplitude, other_direction, other_sharpness):
        ins = [_c(t) for t in (amplitude, direction, sharpness, other_amplitude, other_direction, other_sharpness)]
        out = forward_sg_inner_product(*ins)
        ctx.save_for_backward(*ins)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        ins = ctx.saved_tensors
        return tuple(backward_sg_inner_product(grad_out.contiguous(), *ins, wants=ctx.needs_input_grad))


def forward_sg_inner_product(a, d, s, oa, od, os_):
    out = torch.empty_like(a)
    _lib.call("dibr_b200_sg_inner_product_forward", a.device, a.shape[0], oa.shape[0], a, d, s, oa, od, os_, out)
    return out


def backward_sg_inner_product(grad_out, a, d, s, oa, od, os_, wants=(True,) * 6):
    """-> [grad_amplitude, grad_direction, grad_sharpness, grad_other_*]; None where not wanted."""
    grads = [torch.empty_like(t) if w else None for t, w in zip((a, d, s, oa, od, os_), wants)]
    dev = a.device
    ws = _lib.scratch(_lib.lib().dibr_b200_sg_inner_product_workspace_bytes(oa.shape[0]) if any(wants[3:]) else 0, dev)
    _lib.call("dibr_b200_sg_inner_product_backward", dev,
              a.shape[0], oa.shape[0], grad_out, a, d, s, oa, od, os_, *grads, ws, ws.numel())
    return grads


class DiffuseB200(Function):
    """One shading model (_lib.LIGHT_*) of N points under L lights; albedo may be None."""

    @staticmethod
    def forward(ctx, model, amplitude, direction, sharpness, normal, albedo):
        amplitude, direction, sharpness, normal, albedo = (_c(t) for t in (amplitude, direction, sharpness,
                                                                           normal, albedo))
        N = normal.shape[0]
        L = 1 if model == _lib.LIGHT_SH9 else amplitude.shape[0]
        shape = (N,) if (model == _lib.LIGHT_SH9 and albedo is None) else (N, 3)
        out = torch.empty(shape, dtype=torch.float32, device=normal.device)
        _lib.call("dibr_b200_diffuse_forward", normal.device,
                  model, N, L, amplitude, direction, sharpness, normal, albedo, out)
        ctx.model, ctx.L = model, L
        ctx.save_for_backward(amplitude, direction, sharpness, normal, albedo)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        amplitude, direction, sharpness, normal, albedo = ctx.saved_tensors
        _, w_amp, w_dir, w_sharp, w_n, w_al = ctx.needs_input_grad
        dev = normal.device
        new = lambda t, w: torch.empty_like(t) if (w and t is not None) else None
        g_amp, g_dir, g_sharp = new(amplitude, w_amp), new(direction, w_dir), new(sharpness, w_sharp)
        g_n, g_al = new(normal, w_n), new(albedo, w_al)
        wants_light = any(g is not None for g in (g_amp, g_dir, g_sharp))
        ws = _lib.scratch(_lib.lib().dibr_b200_diffuse_workspace_bytes(ctx.model, ctx.L) if wants_light else 0, dev)
        _lib.call("dibr_b200_diffuse_backward", dev,
                  ctx.model, normal.shape[0], ctx.L, amplitude, direction, sharpness, normal, albedo,
                  grad_out.contiguous(), g_n, g_al, g_amp, g_dir, g_sharp, ws, ws.numel())
        return None, g_amp, g_dir, g_sharp, g_n, g_al


def _check_lights(func, amplitude, direction, sharpness, normal, albedo=None):
    assert amplitude.ndim == 2 and amplitude.shape[1] == 3
    assert direction.shape == amplitude.shape
    assert sharpness.shape == amplitude.shape[:1]
    assert normal.ndim == 2 and normal.shape[1] == 3
    if albedo is not None:
        assert albedo.shape == normal.shape
    _host.check_tensors(func, [("amplitude", amplitude), ("direction", direction), ("sharpness", sharpness),
                               ("normal", normal), ("albedo", albedo)])


def unbatched_reduced_sg_inner_product(amplitude, direction, sharpness,
                                       other_amplitude, other_direction, other_sharpness):
    r"""Fused ``unbatched_sg_inner_product(...).sum(1)``: for every sg of the left-hand side
    (amplitude, direction (num_sg, 3), sharpness (num_sg,)) the sum of its inner products with every
    sg of the right-hand side (num_other, 3), (num_other, 3), (num_other,).  Returns (num_sg, 3).
    Gradients flow to all six inputs; the right-hand side's are bit-reproducible."""
    assert amplitude.ndim == 2 and amplitude.shape[1] == 3
    assert direction.shape == amplitude.shape
    assert sharpness.shape == amplitude.shape[:1]
    assert other_amplitude.ndim == 2 and other_amplitude.shape[1] == 3
    assert other_direction.shape == other_amplitude.shape
    assert other_sharpness.shape == other_amplitude.shape[:1]
    _host.check_tensors("unbatched_reduced_sg_inner_product", [
        ("amplitude", amplitude), ("direction", direction), ("sharpness", sharpness),
        ("other_amplitude", other_amplitude), ("other_direction", other_direction),
        ("other_sharpness", other_sharpness)])
    return UnbatchedReducedSgInnerProductB200.apply(amplitude, direction, sharpness,
                                                    other_amplitude, other_direction, other_sharpness)


def sg_irradiance_inner_product(amplitude, direction, sharpness, normal):
    r"""Irradiance (num_points, 3) at surface points of normal ``normal`` (num_points, 3) from spherical
    Gaussian lights (amplitude, direction (num_sg, 3), sharpness (num_sg,)): the clamped cosine lobe
    approximated as a spherical Gaussian, its inner product with every light, summed and clamped at 0."""
    _check_lights("sg_irradiance_inner_product", amplitude, direction, sharpness, normal)
    return DiffuseB200.apply(_lib.LIGHT_SG_INNER_PRODUCT, amplitude, direction, sharpness, normal, None)


def sg_diffuse_inner_product(amplitude, direction, sharpness, normal, albedo):
    r"""Lambertian outgoing radiance (num_points, 3): ``sg_irradiance_inner_product(...) * albedo / pi``
    (the diffuse term of DIB-R++)."""
    _check_lights("sg_diffuse_inner_product", amplitude, direction, sharpness, normal, albedo)
    return DiffuseB200.apply(_lib.LIGHT_SG_INNER_PRODUCT, amplitude, direction, sharpness, normal, albedo)


def sg_diffuse_fitted(amplitude, direction, sharpness, normal, albedo):
    r"""Lambertian outgoing radiance (num_points, 3) with Stephen Hill's fitted SG irradiance: the mean
    over the lights, clamped at 0, times ``albedo / pi``.  With no light it returns zeros (the
    reference's mean over an empty set is NaN)."""
    _check_lights("sg_diffuse_fitted", amplitude, direction, sharpness, normal, albedo)
    return DiffuseB200.apply(_lib.LIGHT_SG_FITTED, amplitude, direction, sharpness, normal, albedo)


class SpecularB200(Function):
    """sg_warp_specular_term of N points under L lights."""

    @staticmethod
    def forward(ctx, amplitude, direction, sharpness, normal, roughness, view, spec_albedo):
        ins = [_c(t) for t in (amplitude, direction, sharpness, normal, roughness, view, spec_albedo)]
        out = torch.empty_like(ins[3])
        _lib.call("dibr_b200_specular_forward", out.device, out.shape[0], ins[0].shape[0], *ins, out)
        ctx.save_for_backward(*ins)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        ins = ctx.saved_tensors
        wants = ctx.needs_input_grad
        grads = [torch.empty_like(t) if w else None for t, w in zip(ins, wants)]
        dev = ins[3].device
        ws = _lib.scratch(_lib.lib().dibr_b200_specular_workspace_bytes(ins[0].shape[0]) if any(wants[:3]) else 0, dev)
        g_amp, g_dir, g_sharp, g_n, g_r, g_v, g_s = grads
        _lib.call("dibr_b200_specular_backward", dev,
                  ins[3].shape[0], ins[0].shape[0], *ins, grad_out.contiguous(),
                  g_n, g_r, g_v, g_s, g_amp, g_dir, g_sharp, ws, ws.numel())
        return tuple(grads)


def sg_distribution_term(direction, roughness):
    r"""One spherical Gaussian approximating the GGX (Trowbridge-Reitz) normal distribution around
    ``direction`` (num_points, 3) for ``roughness`` (num_points,): with m2 = roughness^2, amplitude
    1 / (pi m2) in each of the three channels (num_points, 3), the input direction, and sharpness
    2 / m2 (num_points,)."""
    assert direction.ndim == 2 and direction.shape[-1]
    assert roughness.shape == direction.shape[:1]
    m2 = roughness * roughness
    amplitude = (1. / (math.pi * m2))[:, None].expand(-1, 3)
    return amplitude, direction, 2. / m2


def _dot(a, b):
    return (a * b).sum(-1)


def sg_warp_distribution(amplitude, direction, sharpness, view):
    r"""The distribution lobe (amplitude, direction (num_sg, 3), sharpness (num_sg,)) turned towards
    the slice of the BRDF seen from ``view`` (num_sg, 3) by Wang et al.'s warp: the direction is the
    reflection of -view about ``direction``, and the sharpness is divided by 4 max(direction . view,
    1e-4).  The amplitude is returned as it is."""
    assert amplitude.ndim == 2 and amplitude.shape[-1] == 3
    assert direction.shape == amplitude.shape
    assert sharpness.shape == amplitude.shape[:1]
    assert view.shape == amplitude.shape
    incoming = -view
    warped = incoming - (2 * _dot(incoming, direction))[:, None] * direction
    return amplitude, warped, sharpness / (4. * torch.clamp(_dot(direction, view), min=1e-4))


def fresnel(ldh, spec_albedo):
    r"""Schlick's Fresnel term: spec_albedo + (1 - spec_albedo) (1 - ldh)^5."""
    return spec_albedo + (1. - spec_albedo) * torch.pow(1. - ldh, 5)


def sg_warp_specular_term(amplitude, direction, sharpness, normal, roughness, view, spec_albedo):
    r"""Cook-Torrance specular reflectance (num_points, 3) of surface points lit by spherical-Gaussian
    lights (amplitude, direction (num_sg, 3), sharpness (num_sg,)): the GGX distribution of
    ``normal`` (num_points, 3) and ``roughness`` (num_points,) as one spherical Gaussian, warped by
    ``view`` (num_points, 3, towards the camera), its inner product with every light summed, times
    the Smith visibility of the light and view directions, Fresnel with ``spec_albedo``
    (num_points, 3) and n . l, clamped at 0 (the specular term of DIB-R++).  One kernel each way;
    the light gradients are bit-reproducible."""
    assert amplitude.ndim == 2 and amplitude.shape[-1] == 3
    assert direction.shape == amplitude.shape
    assert sharpness.shape == amplitude.shape[:1]
    assert normal.ndim == 2 and normal.shape[-1] == 3
    assert roughness.shape == normal.shape[:1]
    assert view.shape == normal.shape
    assert spec_albedo.shape == normal.shape
    _host.check_tensors("sg_warp_specular_term", [
        ("amplitude", amplitude), ("direction", direction), ("sharpness", sharpness), ("normal", normal),
        ("roughness", roughness), ("view", view), ("spec_albedo", spec_albedo)])
    return SpecularB200.apply(amplitude, direction, sharpness, normal, roughness, view, spec_albedo)
