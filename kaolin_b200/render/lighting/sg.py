"""Spherical-Gaussian diffuse lighting — drop-ins for kaolin.render.lighting.sg
(``unbatched_reduced_sg_inner_product``, ``sg_irradiance_inner_product``,
``sg_diffuse_inner_product``, ``sg_diffuse_fitted``).  Each is one sm_90a kernel each way
(kaolin_b200/csrc/lighting.cu) instead of the reference's chains of torch kernels and their
(N, L, 3) temporaries.  Same signatures, shape assertions and return shapes.

Inputs must be float32 CUDA tensors.  The reference's operator is float-only too, but below 8 lights
its torch path would also accept float64; here float64 raises RuntimeError.
"""
import torch
from torch.autograd import Function

from ... import _lib
from ..mesh import _host

__all__ = ["unbatched_reduced_sg_inner_product", "sg_irradiance_inner_product", "sg_diffuse_inner_product",
           "sg_diffuse_fitted"]


def _c(t):
    return None if t is None else t.contiguous()


def _workspace(nbytes, device):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)


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
    dev = a.device
    with torch.cuda.device(dev):
        st = _lib.lib().dibr_b200_sg_inner_product_forward(
            a.shape[0], oa.shape[0], _host.ptr(a), _host.ptr(d), _host.ptr(s), _host.ptr(oa), _host.ptr(od),
            _host.ptr(os_), _host.ptr(out), _host.stream_ptr(dev))
    _lib.check(st, "dibr_b200_sg_inner_product_forward")
    return out


def backward_sg_inner_product(grad_out, a, d, s, oa, od, os_, wants=(True,) * 6):
    """-> [grad_amplitude, grad_direction, grad_sharpness, grad_other_*]; None where not wanted."""
    grads = [torch.empty_like(t) if w else None for t, w in zip((a, d, s, oa, od, os_), wants)]
    dev = a.device
    ws = _workspace(_lib.lib().dibr_b200_sg_inner_product_workspace_bytes(oa.shape[0]) if any(wants[3:]) else 0, dev)
    with torch.cuda.device(dev):
        st = _lib.lib().dibr_b200_sg_inner_product_backward(
            a.shape[0], oa.shape[0], _host.ptr(grad_out), _host.ptr(a), _host.ptr(d), _host.ptr(s), _host.ptr(oa),
            _host.ptr(od), _host.ptr(os_), *[_host.ptr(g) for g in grads], _host.ptr(ws), ws.numel(),
            _host.stream_ptr(dev))
    _lib.check(st, "dibr_b200_sg_inner_product_backward")
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
        with torch.cuda.device(normal.device):
            st = _lib.lib().dibr_b200_diffuse_forward(
                model, N, L, _host.ptr(amplitude), _host.ptr(direction), _host.ptr(sharpness), _host.ptr(normal),
                _host.ptr(albedo), _host.ptr(out), _host.stream_ptr(normal.device))
        _lib.check(st, "dibr_b200_diffuse_forward")
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
        ws = _workspace(_lib.lib().dibr_b200_diffuse_workspace_bytes(ctx.model, ctx.L) if wants_light else 0, dev)
        with torch.cuda.device(dev):
            st = _lib.lib().dibr_b200_diffuse_backward(
                ctx.model, normal.shape[0], ctx.L, _host.ptr(amplitude), _host.ptr(direction), _host.ptr(sharpness),
                _host.ptr(normal), _host.ptr(albedo), _host.ptr(grad_out.contiguous()), _host.ptr(g_n),
                _host.ptr(g_al), _host.ptr(g_amp), _host.ptr(g_dir), _host.ptr(g_sharp), _host.ptr(ws), ws.numel(),
                _host.stream_ptr(dev))
        _lib.check(st, "dibr_b200_diffuse_backward")
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
