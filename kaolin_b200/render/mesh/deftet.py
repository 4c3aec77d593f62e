"""``deftet_sparse_render`` — drop-in for kaolin/render/mesh/deftet.py:269-417 (SURVEY.md §8f rank 3):
the volumetric renderer of DefTet (Gao et al., NeurIPS 2020), which returns ALL intersections of a
list of image points with a mesh, sorted by depth, instead of the closest one.

The two operators run on kaolin_b200/csrc/deftet.cu (uniform-grid face binning, one warp per
point) through ``kaolin_b200._C.render.mesh``; the depth sort, the padding and the feature
interpolation around them are the reference wrapper's own PyTorch glue
(``DeftetSparseRenderer``, deftet.py:269-334).  Same signature, defaults and return structure.
"""
import torch
from torch.autograd import Function

from ... import _C
from . import _host

__all__ = ["deftet_sparse_render"]


class DeftetSparseRendererB200(Function):
    """Counterpart of ``DeftetSparseRenderer`` (deftet.py:269-334)."""

    @staticmethod
    def forward(ctx, pixel_coords, render_ranges, face_vertices_z, face_vertices_image, face_features, knum, eps):
        B, F = face_vertices_z.shape[:2]
        D = face_features.shape[-1]
        P = pixel_coords.shape[1]
        pixel_coords, render_ranges = pixel_coords.contiguous(), render_ranges.contiguous()
        fvz, fvi, ff = face_vertices_z.contiguous(), face_vertices_image.contiguous(), face_features.contiguous()
        bboxes = torch.cat((fvi.min(dim=2)[0], fvi.max(dim=2)[0]), dim=2)
        face_idx, depth, w0, w1 = _C.render.mesh.deftet_sparse_render_forward_cuda(
            fvz, fvi, bboxes, pixel_coords, render_ranges, knum, eps)
        order = torch.argsort(depth, descending=True, dim=-1)
        face_idx = torch.gather(face_idx, -1, order).contiguous()
        w0, w1 = torch.gather(w0, -1, order), torch.gather(w1, -1, order)
        w2 = (face_idx != -1).to(w0.dtype) - (w0 + w1)
        weights = torch.stack([w0, w1, w2], dim=-1).contiguous()
        padded = torch.nn.functional.pad(ff, (0, 0, 0, 0, 1, 0), value=0.)        # face -1 -> a zero face
        sel = torch.gather(padded, 1, (face_idx + 1).reshape(B, -1, 1, 1).expand(B, P * knum, 3, D))
        interpolated = torch.sum(weights.unsqueeze(-1) * sel.reshape(B, P, knum, 3, D), dim=-2).contiguous()
        ctx.save_for_backward(face_idx, weights, fvi, ff)
        ctx.mark_non_differentiable(face_idx)
        ctx.eps = eps
        return interpolated, face_idx

    @staticmethod
    def backward(ctx, grad_interpolated_features, grad_face_idx):
        face_idx, weights, fvi, ff = ctx.saved_tensors
        g_fvi, g_ff = _C.render.mesh.deftet_sparse_render_backward_cuda(
            grad_interpolated_features.contiguous(), face_idx, weights, fvi, ff, ctx.eps)
        return None, None, None, g_fvi, g_ff, None, None


def deftet_sparse_render(pixel_coords, render_ranges, face_vertices_z, face_vertices_image, face_features,
                         knum=300, eps=1e-8):
    r"""Volumetric renderer of DefTet (see kaolin.render.mesh.deftet_sparse_render, deftet.py:337-417).

    Args:
        pixel_coords (B, num_pixels, 2), render_ranges (B, num_pixels, 2),
        face_vertices_z (B, F, 3), face_vertices_image (B, F, 3, 2),
        face_features (B, F, 3, D) or a list of such tensors, knum (default 300), eps (default 1e-8).

    Returns:
        (rendered features (B, num_pixels, knum, D) or a tuple of them, face_idx (B, num_pixels, knum), -1 = void)
    """
    _face_features, split = _host.join_features(face_features)
    image_features, face_idx = DeftetSparseRendererB200.apply(
        pixel_coords, render_ranges, face_vertices_z, face_vertices_image, _face_features, knum, eps)
    return split(image_features), face_idx
