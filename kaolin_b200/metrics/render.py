"""``mask_iou`` — drop-in for kaolin/metrics/render.py:18-41, the silhouette loss the DIB-R loop
applies to the soft mask (SURVEY.md §8f rank 2): the per-view sums of ``lhs*rhs`` and
``lhs+rhs-lhs*rhs`` in one streaming pass and an element-wise backward
(kaolin_b200/csrc/mesh_pipeline.cu) instead of ~8 PyTorch kernels with full-image temporaries."""
import torch
from torch.autograd import Function

from .. import _lib
from ..render.mesh import _host

__all__ = ["mask_iou"]


class MaskIouB200(Function):
    @staticmethod
    def forward(ctx, lhs_mask, rhs_mask):
        l, r = lhs_mask.contiguous(), rhs_mask.contiguous()
        B = l.shape[0]
        hw = l.numel() // B
        sums = torch.empty((B, 2), dtype=torch.float32, device=l.device)
        loss = torch.empty((), dtype=torch.float32, device=l.device)
        _lib.call("dibr_b200_mask_iou_forward", l.device, B, hw, l, r, sums, loss)
        ctx.save_for_backward(l, r, sums)
        return loss

    @staticmethod
    def backward(ctx, g_loss):
        l, r, sums = ctx.saved_tensors
        B = l.shape[0]
        hw = l.numel() // B
        g_l = torch.empty_like(l) if ctx.needs_input_grad[0] else None
        g_r = torch.empty_like(r) if ctx.needs_input_grad[1] else None
        g = g_loss.contiguous().to(torch.float32)
        _lib.call("dibr_b200_mask_iou_backward", l.device, B, hw, l, r, sums, g, g_l, g_r)
        return g_l, g_r


def mask_iou(lhs_mask, rhs_mask):
    r"""IoU loss of two segmentation masks of shape (batch_size, height, width):
    ``1 - mean_b( sum(l*r) / (sum(l + r - l*r) + 1e-10) )`` (kaolin.metrics.render.mask_iou).

    Either mask may be a ``bool`` or integer tensor (``target > 0.5``, ``face_idx >= 0``): it is
    converted to float32, as the reference's type promotion against a float mask does, and gets no
    gradient.  A floating mask must be float32; float16, bfloat16 and float64 raise RuntimeError.
    Nothing clamps the values: masks outside [0, 1] enter the sums as they are.  A view whose
    union is empty contributes an IoU of 0 (the ``1e-10``), so two empty batches give a loss of
    exactly 1 and zero gradients.  At most 65535 views per call."""
    _host.check_tensors("mask_iou", [("lhs_mask", lhs_mask), ("rhs_mask", rhs_mask)])
    if lhs_mask.dim() != 3:
        raise RuntimeError("mask_iou: masks must be of shape (batch_size, height, width)")
    assert rhs_mask.shape == lhs_mask.shape
    if lhs_mask.shape[0] > 65535:
        raise RuntimeError(f"mask_iou: at most 65535 views per call, got {lhs_mask.shape[0]}")
    lhs_mask, rhs_mask = (m if m.is_floating_point() or m.is_complex() else m.to(torch.float32)
                          for m in (lhs_mask, rhs_mask))
    _host.check_float32("mask_iou", [("lhs_mask", lhs_mask), ("rhs_mask", rhs_mask)])
    return MaskIouB200.apply(lhs_mask, rhs_mask)
