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
    """Counterpart of ``DibrSoftMaskCuda`` (dibr.py:27-73), in float32 or float64.  The K-lists
    the reference saves (13*knum bytes per pixel) are recomputed in backward."""

    @staticmethod
    def forward(ctx, face_vertices_image, selected_face_idx, sigmainv, boxlen, knum, multiplier):
        fvi = face_vertices_image.contiguous()
        idx = selected_face_idx.contiguous()
        B, H, W = idx.shape
        boxlen_m = boxlen * multiplier          # a Python float: double, as dibr.py:36-37
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


def dibr_soft_mask(face_vertices_image, selected_face_idx, sigmainv=7000, boxlen=0.02,
                   knum=30, multiplier=1000.):
    r"""Soft mask of DIB-R (see kaolin.render.mesh.dibr_soft_mask, dibr.py:75-117); float64
    vertices run it in float64."""
    f64 = _host.any_double(face_vertices_image)
    _host.check_tensors("dibr_soft_mask", [("face_vertices_image", face_vertices_image),
                                           ("selected_face_idx", selected_face_idx)],
                        dtype=None if f64 else torch.float32)
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
    """rasterize(valid = face_normals_z >= 0) + dibr_soft_mask in one node, in float32 / bf16
    features or float64."""

    @staticmethod
    def forward(ctx, height, width, face_vertices_z, face_vertices_image, face_features,
                face_normals_z, sigmainv, boxlen, knum, multiplier, eps, soft_multiplier):
        fvz = face_vertices_z.contiguous()
        fvi = face_vertices_image.contiguous()
        ff = face_features.contiguous()
        fnz = face_normals_z.contiguous()
        boxlen_m = boxlen * soft_multiplier
        feat, face_idx, wts, soft, ws = _host.forward(
            _lib.RASTER | _lib.SOFT_MASK, height, width, fvz, fvi, ff, fnz, None,
            multiplier, eps, sigmainv, boxlen_m, knum)
        ctx.save_for_backward(face_idx, wts, soft, fvi, ff)
        ctx.mark_non_differentiable(face_idx)
        ctx.set_materialize_grads(False)   # no 8 B/pixel zero "gradient" for face_idx
        ctx.params = (height, width, multiplier, eps, sigmainv, boxlen_m, knum)
        # inference / no_grad callers do not pin the workspace (bins + hit cache) until the graph dies
        ctx.ws = ws if (ctx.needs_input_grad[3] or ctx.needs_input_grad[4]) else None
        return feat, soft, face_idx

    @staticmethod
    def backward(ctx, grad_features, grad_soft_mask, grad_face_idx):
        face_idx, wts, soft, fvi, ff = ctx.saved_tensors
        height, width, multiplier, eps, sigmainv, boxlen_m, knum = ctx.params
        g_feat = None if grad_features is None else grad_features.contiguous()
        g_soft = None if grad_soft_mask is None else grad_soft_mask.contiguous()
        pipe = getattr(ctx, "view_pipeline", None)      # set on this node by PipelinedGradAllGather.attach
        if pipe is not None and g_feat is not None and g_soft is not None and ctx.ws is not None \
                and fvi.dtype != torch.float64:          # the float64 backward is one kernel: no view chunks
            # backward in view chunks; the exchange of chunk i travels while chunk i+1 computes
            g_fvi = torch.empty_like(fvi)
            g_ff = torch.empty(ff.shape, dtype=torch.float32, device=ff.device)

            def run_chunk(c0, c1, hook):
                _host.backward(height, width, g_feat, g_soft, face_idx, None, soft, fvi, ff, multiplier, eps, sigmainv,
                               boxlen_m, knum, ctx.ws, True, feature_grad_hook=hook, views=(c0, c1), out=(g_fvi, g_ff))
            pipe(fvi.shape[0], run_chunk, g_fvi, g_ff)
            return None, None, None, g_fvi, g_ff.to(ff.dtype), None, None, None, None, None, None, None
        # per-node hook (set on this node by OverlappedGradAllGather.attach, never global)
        g_fvi, g_ff = _host.backward(height, width, g_feat, g_soft, face_idx, wts, soft, fvi, ff,
                                     multiplier, eps, sigmainv, boxlen_m, knum, ctx.ws, ctx.ws is not None,
                                     feature_grad_hook=getattr(ctx, "feature_grad_hook", None))
        g_ff = g_ff.to(ff.dtype)      # fp32 accumulation; autograd wants the input's dtype (bf16 features)
        return None, None, None, g_fvi, g_ff, None, None, None, None, None, None, None


def dibr_rasterization(height, width, face_vertices_z, face_vertices_image, face_features,
                       face_normals_z, sigmainv=7000, boxlen=0.02, knum=30, multiplier=None,
                       eps=None, rast_backend='cuda'):
    r"""Fully differentiable DIB-R renderer (see kaolin.render.mesh.dibr_rasterization,
    dibr.py:119-209): returns (interpolated_features | tuple, soft_mask, face_idx).  A float64
    input among the vertices, features and normals runs the whole call in float64."""
    if rast_backend != 'cuda':
        raise ValueError(f'"{rast_backend}" is not a valid backend, '
                         'kaolin_b200 only provides ["cuda"]')
    if multiplier is None:
        multiplier = 1000
        soft_multiplier = 1000.          # dibr.py:200
    else:
        soft_multiplier = multiplier
    if eps is None:
        eps = 1e-8
    _face_features, split = _host.join_features(face_features)
    f64 = _host.any_double(face_vertices_z, face_vertices_image, face_normals_z, _face_features)
    B, F = _check_inputs("dibr_rasterization", face_vertices_z, face_vertices_image, _face_features, f64)
    _host.check_tensors("dibr_rasterization", [("face_vertices_z", face_vertices_z),
                                               ("face_normals_z", face_normals_z)],
                        dtype=None if f64 else torch.float32)
    _host.check_size("dibr_rasterization", "face_normals_z", face_normals_z, (B, F))
    if f64:      # cast here, not in the Function: autograd returns each input's gradient in its own dtype
        face_vertices_z, face_vertices_image, _face_features, face_normals_z = (
            t.double() for t in (face_vertices_z, face_vertices_image, _face_features, face_normals_z))
    image_features, soft_mask, face_idx = DibrRasterizationB200.apply(
        height, width, face_vertices_z, face_vertices_image, _face_features, face_normals_z,
        sigmainv, boxlen, knum, multiplier, eps, soft_multiplier)
    return split(image_features), soft_mask, face_idx
