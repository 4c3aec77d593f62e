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
    """Counterpart of ``RasterizeCuda`` (rasterization.py:226-371), in float32 / bf16 features or,
    as the reference dispatches float and double, in float64 (the reference's <double> arithmetic)."""

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
        feat, face_idx, wts, _, _ = _host.forward(
            _lib.RASTER, height, width, fvz, fvi, ff, None, valid_u8, multiplier, eps, 0., 0., 0)
        ctx.save_for_backward(face_idx, wts, fvi, ff)
        ctx.mark_non_differentiable(face_idx)
        ctx.set_materialize_grads(False)   # no 8 B/pixel zero "gradient" for face_idx
        ctx.multiplier = multiplier        # the backward recomputes the weights with it
        ctx.eps = eps
        ctx.hw = (height, width)
        return feat, face_idx

    @staticmethod
    def backward(ctx, grad_interpolated_features, grad_face_idx):
        if grad_interpolated_features is None:      # no gradient reached the features (grads not materialized)
            return None, None, None, None, None, None, None, None
        face_idx, wts, fvi, ff = ctx.saved_tensors
        g = grad_interpolated_features.contiguous()
        # float64 stores the weights and reads them back: the multiplier is not used then
        multiplier = ctx.multiplier if wts is None else 1.0
        g_fvi, g_ff = _host.backward(ctx.hw[0], ctx.hw[1], g, None, face_idx, wts, None, fvi, ff,
                                     multiplier, ctx.eps, 0., 0., 0, None, False)
        g_ff = g_ff.to(ff.dtype)      # fp32 accumulation; autograd wants the input's dtype (bf16 features)
        # the reference never produces a gradient for face_vertices_z (rasterization.py:370-371)
        return None, None, None, g_fvi, g_ff, None, None, None


def _check_inputs(func, face_vertices_z, face_vertices_image, face_features, f64):
    """Device and shape checks; float64 calls accept any dtype, which the caller casts to double."""
    _host.check_tensors(func, [("face_vertices_z", face_vertices_z),
                               ("face_vertices_image", face_vertices_image)],
                        dtype=None if f64 else torch.float32)
    _host.check_tensors(func, [("face_vertices_z", face_vertices_z), ("face_features", face_features)],
                        dtype=None)                       # same device; the dtype is checked next
    if not f64:
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
    Only ``backend='cuda'`` exists here (no multi-backend dispatch).  A float64 input among
    the vertices and features runs the whole call in float64.
    """
    if multiplier is None:
        multiplier = 1000
    if eps is None:
        eps = 1e-8
    if backend != 'cuda':
        raise ValueError(f'"{backend}" is not a valid backend, '
                         'kaolin_b200 only provides ["cuda"]')
    _face_features, split = _host.join_features(face_features)
    f64 = _host.any_double(face_vertices_z, face_vertices_image, _face_features)
    B, F = _check_inputs("rasterize", face_vertices_z, face_vertices_image, _face_features, f64)
    if valid_faces is not None:
        _host.check_tensors("rasterize", [("face_vertices_z", face_vertices_z),
                                          ("valid_faces", valid_faces)], dtype=None)
        _host.check_size("rasterize", "valid_faces", valid_faces, (B, F))
    if f64:      # cast here, not in the Function: autograd returns each input's gradient in its own dtype
        face_vertices_z, face_vertices_image, _face_features = (
            t.double() for t in (face_vertices_z, face_vertices_image, _face_features))
    image_features, face_idx = RasterizeB200.apply(
        height, width, face_vertices_z, face_vertices_image, _face_features, valid_faces,
        multiplier, eps)
    return split(image_features), face_idx
