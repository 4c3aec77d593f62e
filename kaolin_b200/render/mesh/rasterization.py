"""``rasterize`` — drop-in for kaolin/render/mesh/rasterization.py:373-492 (backend 'cuda').

Same signature, defaults, return structure and dtypes as the reference; the
valid-face packing, multiplier scaling, bbox construction and index remapping the
reference does with ~12 PyTorch kernels (rasterization.py:290-346) happen inside
the sm_90a kernels behind ``dibr_b200_forward`` (include/dibr_b200.h).
"""
import torch
from torch.autograd import Function

from ... import _lib
from . import _host

__all__ = ["rasterize"]


class RasterizeB200(Function):
    """Counterpart of ``RasterizeCuda`` (rasterization.py:226-371)."""

    @staticmethod
    def forward(ctx, height, width, face_vertices_z, face_vertices_image, face_features,
                valid_faces, multiplier, eps):
        fvz = face_vertices_z.contiguous()
        fvi = face_vertices_image.contiguous()
        ff = face_features.contiguous()
        valid_u8 = None
        if valid_faces is not None:
            valid_u8 = valid_faces.contiguous()
            valid_u8 = valid_u8.view(torch.uint8) if valid_u8.dtype == torch.bool else valid_u8.ne(0).view(torch.uint8)
        feat, face_idx, _, _, _ = _host.forward(
            _lib.RASTER, height, width, fvz, fvi, ff, None, valid_u8, multiplier, eps, 0., 0., 0)
        ctx.save_for_backward(face_idx, fvi, ff)
        ctx.mark_non_differentiable(face_idx)
        ctx.set_materialize_grads(False)   # no 8 B/pixel zero "gradient" for face_idx
        ctx.multiplier = multiplier        # the backward recomputes the weights with it
        ctx.eps = eps
        ctx.hw = (height, width)
        return feat, face_idx

    @staticmethod
    def backward(ctx, grad_interpolated_features, grad_face_idx):
        face_idx, fvi, ff = ctx.saved_tensors
        g = grad_interpolated_features.contiguous()
        g_fvi, g_ff = _host.backward(ctx.hw[0], ctx.hw[1], g, None, face_idx, None, None, fvi, ff,
                                     ctx.multiplier, ctx.eps, 0., 0., 0, None, False)
        g_ff = g_ff.to(ff.dtype)      # fp32 accumulation; autograd wants the input's dtype (bf16 features)
        # the reference never produces a gradient for face_vertices_z (rasterization.py:370-371)
        return None, None, None, g_fvi, g_ff, None, None, None


class RasterizeF64(Function):
    """float64 instantiation of ``RasterizeCuda`` (the reference dispatches float and double):
    dibr_b200_forward_f64 / dibr_b200_backward_f64, the reference's <double> arithmetic."""

    @staticmethod
    def forward(ctx, height, width, fvz, fvi, ff, valid_faces, multiplier, eps):
        fvz, fvi, ff = fvz.contiguous(), fvi.contiguous(), ff.contiguous()
        valid_u8 = None
        if valid_faces is not None:
            valid_u8 = valid_faces.contiguous()
            valid_u8 = valid_u8.view(torch.uint8) if valid_u8.dtype == torch.bool else valid_u8.ne(0).view(torch.uint8)
        feat, face_idx, wts, _, _ = _host.forward_f64(_lib.RASTER, height, width, fvz, fvi, ff, None, valid_u8,
                                                      multiplier, eps, 0., 0., 0)
        ctx.save_for_backward(face_idx, wts, fvi, ff)
        ctx.mark_non_differentiable(face_idx)
        ctx.args = (height, width, eps)
        return feat, face_idx

    @staticmethod
    def backward(ctx, grad_interpolated_features, grad_face_idx):
        face_idx, wts, fvi, ff = ctx.saved_tensors
        height, width, eps = ctx.args
        g_fvi, g_ff = _host.backward_f64(height, width, grad_interpolated_features.contiguous(), None, face_idx, wts,
                                         None, fvi, ff, 1.0, eps, 0., 0., 0, None)
        return None, None, None, g_fvi, g_ff, None, None, None


def _rasterize_f64(height, width, face_vertices_z, face_vertices_image, face_features, valid_faces, multiplier, eps):
    is_list = isinstance(face_features, (list, tuple))
    ff = torch.cat(face_features, dim=-1) if is_list else face_features
    d = torch.float64
    tensors = [("face_vertices_z", face_vertices_z), ("face_vertices_image", face_vertices_image),
               ("face_features", ff)]
    _host.check_tensors("rasterize", tensors, dtype=None)
    if face_vertices_z.dim() != 3 or face_vertices_z.shape[-1] != 3:
        raise RuntimeError("rasterize: face_vertices_z must be of shape (batch_size, num_faces, 3)")
    B, F, _ = face_vertices_z.shape
    _host.check_size("rasterize", "face_vertices_image", face_vertices_image, (B, F, 3, 2))
    _host.check_size("rasterize", "face_features", ff, (B, F, 3, ff.shape[-1]))
    out, face_idx = RasterizeF64.apply(height, width, face_vertices_z.to(d), face_vertices_image.to(d), ff.to(d),
                                       valid_faces, multiplier, eps)
    if is_list:
        outs, cur = [], 0
        for f in face_features:
            outs.append(out[..., cur:cur + f.shape[-1]])
            cur += f.shape[-1]
        out = tuple(outs)
    return out, face_idx


def _check_inputs(func, face_vertices_z, face_vertices_image, face_features):
    _host.check_tensors(func, [("face_vertices_z", face_vertices_z),
                               ("face_vertices_image", face_vertices_image)])
    _host.check_tensors(func, [("face_vertices_z", face_vertices_z), ("face_features", face_features)],
                        dtype=None)                       # same device; the dtype is checked next
    _host.check_feature_dtype(func, "face_features", face_features)
    if face_vertices_z.dim() != 3 or face_vertices_z.shape[-1] != 3:
        raise RuntimeError(f"{func}: face_vertices_z must be of shape (batch_size, num_faces, 3)")
    B, F, _ = face_vertices_z.shape
    _host.check_size(func, "face_vertices_image", face_vertices_image, (B, F, 3, 2))
    if face_features.dim() != 4:
        raise RuntimeError(f"{func}: face_features must be of shape (batch_size, num_faces, 3, feature_dim)")
    _host.check_size(func, "face_features", face_features, (B, F, 3, face_features.shape[-1]))
    return B, F


def rasterize(height, width, face_vertices_z, face_vertices_image, face_features,
              valid_faces=None, multiplier=None, eps=None, backend='cuda'):
    r"""Fully differentiable rasterization (see kaolin.render.mesh.rasterize).

    Args and returns are those of the reference (rasterization.py:393-453).
    Only ``backend='cuda'`` exists here (no multi-backend dispatch).
    """
    if multiplier is None:
        multiplier = 1000
    if eps is None:
        eps = 1e-8
    if backend != 'cuda':
        raise ValueError(f'"{backend}" is not a valid backend, '
                         'kaolin_b200 only provides ["cuda"]')
    flat = list(face_features) if isinstance(face_features, (list, tuple)) else [face_features]
    if any(isinstance(t, torch.Tensor) and t.dtype == torch.float64
           for t in (face_vertices_z, face_vertices_image, *flat)):
        return _rasterize_f64(height, width, face_vertices_z, face_vertices_image, face_features, valid_faces,
                              multiplier, eps)
    _face_features = torch.cat(face_features, dim=-1) \
        if isinstance(face_features, (list, tuple)) else face_features
    B, F = _check_inputs("rasterize", face_vertices_z, face_vertices_image, _face_features)
    if valid_faces is not None:
        _host.check_tensors("rasterize", [("face_vertices_z", face_vertices_z),
                                          ("valid_faces", valid_faces)], dtype=None)
        _host.check_size("rasterize", "valid_faces", valid_faces, (B, F))
    image_features, face_idx = RasterizeB200.apply(
        height, width, face_vertices_z, face_vertices_image, _face_features, valid_faces,
        multiplier, eps)
    if isinstance(face_features, (list, tuple)):
        _image_features = []
        cur_idx = 0
        for face_feature in face_features:
            _image_features.append(image_features[..., cur_idx:cur_idx + face_feature.shape[-1]])
            cur_idx += face_feature.shape[-1]
        image_features = tuple(_image_features)
    return image_features, face_idx
