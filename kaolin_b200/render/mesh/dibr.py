"""``dibr_soft_mask`` / ``dibr_rasterization`` — drop-in for kaolin/render/mesh/dibr.py.

``dibr_rasterization`` is ONE autograd node: the forward is a single fused tile
kernel (rasterize + soft mask share the face binning), the backward adds the
rasterize and soft-mask gradients of ``face_vertices_image`` in place of the
reference's two nodes + autograd sum (SURVEY.md §3.2).  Results are identical to
calling ``rasterize`` then ``dibr_soft_mask``
(tests/test_parity_gpu.py::test_composition_equals_separate_calls).
"""
import torch
from torch.autograd import Function

from ... import _lib
from . import _host
from .rasterization import _check_inputs

__all__ = ["dibr_soft_mask", "dibr_rasterization"]


class DibrSoftMaskB200(Function):
    """Counterpart of ``DibrSoftMaskCuda`` (dibr.py:27-73).  The K-lists the
    reference saves (13*knum bytes per pixel) are recomputed in backward."""

    @staticmethod
    def forward(ctx, face_vertices_image, selected_face_idx, sigmainv, boxlen, knum, multiplier):
        fvi = face_vertices_image.contiguous()
        idx = selected_face_idx.contiguous()
        B, H, W = idx.shape
        boxlen_m = boxlen * multiplier
        _, _, _, soft, ws = _host.forward(_lib.SOFT_MASK, H, W, None, fvi, None, None, None,
                                          multiplier, 0., sigmainv, boxlen_m, knum, face_idx_in=idx)
        ctx.save_for_backward(soft, fvi, idx)
        ctx.params = (sigmainv, boxlen_m, knum, multiplier)
        # the workspace (bins + hit cache, up to CACHE_MAX_BYTES) is only worth keeping for a backward
        ctx.ws = ws if ctx.needs_input_grad[0] else None      # (grad mode is off inside forward: do not test it)
        return soft

    @staticmethod
    def backward(ctx, grad_soft_mask):
        soft, fvi, idx = ctx.saved_tensors
        sigmainv, boxlen_m, knum, multiplier = ctx.params
        B, H, W = idx.shape
        g_fvi, _ = _host.backward(H, W, None, grad_soft_mask.contiguous(), idx, None, soft, fvi, None,
                                  multiplier, 0., sigmainv, boxlen_m, knum, ctx.ws, ctx.ws is not None)
        return g_fvi, None, None, None, None, None


class DibrSoftMaskF64(Function):
    """float64 instantiation of ``DibrSoftMaskCuda`` (dibr_b200_forward_f64, mode SOFT_MASK)."""

    @staticmethod
    def forward(ctx, face_vertices_image, selected_face_idx, sigmainv, boxlen, knum, multiplier):
        fvi, idx = face_vertices_image.contiguous(), selected_face_idx.contiguous()
        B, H, W = idx.shape
        boxlen_m = boxlen * multiplier                                    # a Python float: double, as dibr.py:36-37
        _, _, _, soft, ws = _host.forward_f64(_lib.SOFT_MASK, H, W, None, fvi, None, None, None, multiplier, 0.,
                                              sigmainv, boxlen_m, knum, face_idx_in=idx)
        ctx.save_for_backward(soft, fvi, idx)
        ctx.params = (sigmainv, boxlen_m, knum, multiplier)
        ctx.ws = ws if ctx.needs_input_grad[0] else None
        return soft

    @staticmethod
    def backward(ctx, grad_soft_mask):
        soft, fvi, idx = ctx.saved_tensors
        sigmainv, boxlen_m, knum, multiplier = ctx.params
        B, H, W = idx.shape
        g_fvi, _ = _host.backward_f64(H, W, None, grad_soft_mask.contiguous(), idx, None, soft, fvi, None, multiplier,
                                      0., sigmainv, boxlen_m, knum, ctx.ws)
        return g_fvi, None, None, None, None, None


class DibrRasterizationF64(Function):
    """float64 instantiation of the fused node (the reference's <double> kernels' arithmetic)."""

    @staticmethod
    def forward(ctx, height, width, fvz, fvi, ff, fnz, sigmainv, boxlen, knum, multiplier, eps, soft_multiplier):
        fvz, fvi, ff, fnz = fvz.contiguous(), fvi.contiguous(), ff.contiguous(), fnz.contiguous()
        boxlen_m = boxlen * soft_multiplier
        feat, face_idx, wts, soft, ws = _host.forward_f64(_lib.RASTER | _lib.SOFT_MASK, height, width, fvz, fvi, ff,
                                                          fnz, None, multiplier, eps, sigmainv, boxlen_m, knum)
        ctx.save_for_backward(face_idx, wts, soft, fvi, ff)
        ctx.mark_non_differentiable(face_idx)
        ctx.set_materialize_grads(False)
        ctx.params = (height, width, multiplier, eps, sigmainv, boxlen_m, knum)
        ctx.ws = ws if (ctx.needs_input_grad[3] or ctx.needs_input_grad[4]) else None
        return feat, soft, face_idx

    @staticmethod
    def backward(ctx, grad_features, grad_soft_mask, grad_face_idx):
        face_idx, wts, soft, fvi, ff = ctx.saved_tensors
        height, width, multiplier, eps, sigmainv, boxlen_m, knum = ctx.params
        g_feat = None if grad_features is None else grad_features.contiguous()
        g_soft = None if grad_soft_mask is None else grad_soft_mask.contiguous()
        g_fvi, g_ff = _host.backward_f64(height, width, g_feat, g_soft, face_idx, wts, soft, fvi, ff, multiplier, eps,
                                         sigmainv, boxlen_m, knum, ctx.ws)
        # per-node hook of the multi-GPU gathers (multi_gpu.*.attach); the float64 backward is one kernel, so the
        # feature gradient is handed over at the end instead of between the branches
        hook = getattr(ctx, "feature_grad_hook", None)
        if hook is not None and g_feat is not None and g_soft is not None:
            hook(g_ff)
        return None, None, None, g_fvi, g_ff, None, None, None, None, None, None, None


def _dibr_rasterization_f64(height, width, face_vertices_z, face_vertices_image, face_features, face_normals_z,
                            sigmainv, boxlen, knum, multiplier, eps):
    if multiplier is None:
        multiplier, soft_multiplier = 1000, 1000.
    else:
        soft_multiplier = multiplier
    if eps is None:
        eps = 1e-8
    is_list = isinstance(face_features, (list, tuple))
    ff = torch.cat(face_features, dim=-1) if is_list else face_features
    _host.check_tensors("dibr_rasterization", [("face_vertices_z", face_vertices_z),
                                               ("face_vertices_image", face_vertices_image), ("face_features", ff),
                                               ("face_normals_z", face_normals_z)], dtype=None)
    if face_vertices_z.dim() != 3 or face_vertices_z.shape[-1] != 3:
        raise RuntimeError("dibr_rasterization: face_vertices_z must be of shape (batch_size, num_faces, 3)")
    B, F, _ = face_vertices_z.shape
    _host.check_size("dibr_rasterization", "face_vertices_image", face_vertices_image, (B, F, 3, 2))
    _host.check_size("dibr_rasterization", "face_features", ff, (B, F, 3, ff.shape[-1]))
    _host.check_size("dibr_rasterization", "face_normals_z", face_normals_z, (B, F))
    d = torch.float64
    feat, soft, face_idx = DibrRasterizationF64.apply(
        height, width, face_vertices_z.to(d), face_vertices_image.to(d), ff.to(d), face_normals_z.to(d),
        sigmainv, boxlen, knum, multiplier, eps, soft_multiplier)
    if is_list:
        outs, cur = [], 0
        for f in face_features:
            outs.append(feat[..., cur:cur + f.shape[-1]])
            cur += f.shape[-1]
        feat = tuple(outs)
    return feat, soft, face_idx


def dibr_soft_mask(face_vertices_image, selected_face_idx, sigmainv=7000, boxlen=0.02,
                   knum=30, multiplier=1000.):
    r"""Soft mask of DIB-R (see kaolin.render.mesh.dibr_soft_mask, dibr.py:75-117)."""
    if face_vertices_image.dtype == torch.float64:
        _host.check_tensors("dibr_soft_mask", [("face_vertices_image", face_vertices_image),
                                               ("selected_face_idx", selected_face_idx)], dtype=None)
        return DibrSoftMaskF64.apply(face_vertices_image, selected_face_idx, sigmainv, boxlen, knum, multiplier)
    _host.check_tensors("dibr_soft_mask", [("face_vertices_image", face_vertices_image),
                                           ("selected_face_idx", selected_face_idx)])
    if face_vertices_image.dim() != 4 or tuple(face_vertices_image.shape[2:]) != (3, 2):
        raise RuntimeError("dibr_soft_mask: face_vertices_image must be of shape "
                           "(batch_size, num_faces, 3, 2)")
    if selected_face_idx.dtype != torch.int64 or selected_face_idx.dim() != 3 \
            or selected_face_idx.shape[0] != face_vertices_image.shape[0]:
        raise RuntimeError("dibr_soft_mask: selected_face_idx must be a LongTensor of shape "
                           "(batch_size, height, width)")
    return DibrSoftMaskB200.apply(face_vertices_image, selected_face_idx, sigmainv, boxlen,
                                  knum, multiplier)


class DibrRasterizationB200(Function):
    """rasterize(valid = face_normals_z >= 0) + dibr_soft_mask in one node."""

    @staticmethod
    def forward(ctx, height, width, face_vertices_z, face_vertices_image, face_features,
                face_normals_z, sigmainv, boxlen, knum, multiplier, eps, soft_multiplier):
        fvz = face_vertices_z.contiguous()
        fvi = face_vertices_image.contiguous()
        ff = face_features.contiguous()
        fnz = face_normals_z.contiguous()
        boxlen_m = boxlen * soft_multiplier
        feat, face_idx, _, soft, ws = _host.forward(
            _lib.RASTER | _lib.SOFT_MASK, height, width, fvz, fvi, ff, fnz, None,
            multiplier, eps, sigmainv, boxlen_m, knum)
        ctx.save_for_backward(face_idx, soft, fvi, ff)
        ctx.mark_non_differentiable(face_idx)
        ctx.set_materialize_grads(False)   # no 8 B/pixel zero "gradient" for face_idx
        ctx.params = (height, width, multiplier, eps, sigmainv, boxlen_m, knum)
        # inference / no_grad callers do not pin the workspace (bins + hit cache) until the graph dies
        ctx.ws = ws if (ctx.needs_input_grad[3] or ctx.needs_input_grad[4]) else None
        return feat, soft, face_idx

    @staticmethod
    def backward(ctx, grad_features, grad_soft_mask, grad_face_idx):
        face_idx, soft, fvi, ff = ctx.saved_tensors
        height, width, multiplier, eps, sigmainv, boxlen_m, knum = ctx.params
        g_feat = None if grad_features is None else grad_features.contiguous()
        g_soft = None if grad_soft_mask is None else grad_soft_mask.contiguous()
        pipe = getattr(ctx, "view_pipeline", None)      # set on this node by PipelinedGradAllGather.attach
        if pipe is not None and g_feat is not None and g_soft is not None and ctx.ws is not None:
            # backward in view chunks; the exchange of chunk i travels while chunk i+1 computes
            g_fvi = torch.empty_like(fvi)
            g_ff = torch.empty(ff.shape, dtype=torch.float32, device=ff.device)

            def run_chunk(c0, c1, hook):
                _host.backward(height, width, g_feat, g_soft, face_idx, None, soft, fvi, ff, multiplier, eps, sigmainv,
                               boxlen_m, knum, ctx.ws, True, feature_grad_hook=hook, views=(c0, c1), out=(g_fvi, g_ff))
            pipe(fvi.shape[0], run_chunk, g_fvi, g_ff)
            return None, None, None, g_fvi, g_ff.to(ff.dtype), None, None, None, None, None, None, None
        # per-node hook (set on this node by OverlappedGradAllGather.attach, never global)
        g_fvi, g_ff = _host.backward(height, width, g_feat, g_soft, face_idx, None, soft, fvi, ff,
                                     multiplier, eps, sigmainv, boxlen_m, knum, ctx.ws, ctx.ws is not None,
                                     feature_grad_hook=getattr(ctx, "feature_grad_hook", None))
        g_ff = g_ff.to(ff.dtype)      # fp32 accumulation; autograd wants the input's dtype (bf16 features)
        return None, None, None, g_fvi, g_ff, None, None, None, None, None, None, None


def dibr_rasterization(height, width, face_vertices_z, face_vertices_image, face_features,
                       face_normals_z, sigmainv=7000, boxlen=0.02, knum=30, multiplier=None,
                       eps=None, rast_backend='cuda'):
    r"""Fully differentiable DIB-R renderer (see kaolin.render.mesh.dibr_rasterization,
    dibr.py:119-209): returns (interpolated_features | tuple, soft_mask, face_idx)."""
    if rast_backend != 'cuda':
        raise ValueError(f'"{rast_backend}" is not a valid backend, '
                         'kaolin_b200 only provides ["cuda"]')
    flat = list(face_features) if isinstance(face_features, (list, tuple)) else [face_features]
    if any(isinstance(t, torch.Tensor) and t.dtype == torch.float64
           for t in (face_vertices_z, face_vertices_image, face_normals_z, *flat)):
        return _dibr_rasterization_f64(height, width, face_vertices_z, face_vertices_image, face_features,
                                       face_normals_z, sigmainv, boxlen, knum, multiplier, eps)
    if multiplier is None:
        multiplier = 1000
        soft_multiplier = 1000.          # dibr.py:200
    else:
        soft_multiplier = multiplier
    if eps is None:
        eps = 1e-8
    _face_features = torch.cat(face_features, dim=-1) \
        if isinstance(face_features, (list, tuple)) else face_features
    B, F = _check_inputs("dibr_rasterization", face_vertices_z, face_vertices_image, _face_features)
    _host.check_tensors("dibr_rasterization", [("face_vertices_z", face_vertices_z),
                                               ("face_normals_z", face_normals_z)])
    _host.check_size("dibr_rasterization", "face_normals_z", face_normals_z, (B, F))
    image_features, soft_mask, face_idx = DibrRasterizationB200.apply(
        height, width, face_vertices_z, face_vertices_image, _face_features, face_normals_z,
        sigmainv, boxlen, knum, multiplier, eps, soft_multiplier)
    if isinstance(face_features, (list, tuple)):
        _image_features = []
        cur_idx = 0
        for face_feature in face_features:
            _image_features.append(image_features[..., cur_idx:cur_idx + face_feature.shape[-1]])
            cur_idx += face_feature.shape[-1]
        image_features = tuple(_image_features)
    return image_features, soft_mask, face_idx
