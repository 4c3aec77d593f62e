"""kaolin.ops.pointcloud on sm_90a kernels (csrc/pointcloud.cu): ``farthest_point_sampling`` and
``center_points``.

The reference samples with NVIDIA Warp, one view at a time, reads a round counter back to the host,
resolves equal distances through races and returns a CPU tensor.  Here every view goes through one
call with no host read, the result is fixed bit for bit by a stated contract and stays on the
points' device.
"""
import torch

from .. import _lib

__all__ = ["center_points", "farthest_point_sampling"]


def center_points(points, normalize=False, eps=1e-6):
    r"""kaolin.ops.pointcloud.center_points: each view of ``points`` (B, N, C) moved so that the middle of
    its per-channel bounding box is at the origin; with ``normalize``, also divided by the box's longest
    side, clamped below at ``eps``, so the view spans [-0.5, 0.5] along that side.  Same shape, device
    and dtype as the input.

    Plain torch, bit-equal to the reference on every floating dtype (NaN propagates through the box as
    in ``torch.min`` / ``torch.max``).  There is no CPU path: a CPU tensor raises NotImplementedError.
    A tensor that is not 3-dimensional raises ``ValueError`` (the reference asserts).
    """
    if not points.is_cuda:
        raise NotImplementedError("center_points does not support CPU.")
    if points.ndim != 3:
        raise ValueError(f"Points have unexpected shape {tuple(points.shape)}")
    lo, hi = torch.aminmax(points, dim=1, keepdim=True)
    out = points - (lo + hi) / 2
    if normalize:
        out = out / (hi - lo).amax(dim=-1, keepdim=True).clamp(min=eps)
    return out


def farthest_point_sampling(points, k):
    r"""kaolin.ops.pointcloud.farthest_point_sampling: for each view of ``points`` (B, N, 3) float32 on a
    CUDA device, the indices of ``k`` points, each the farthest from those taken before it, as int64
    (B, k) on the points' device.  ``0 <= k <= N``.

    The output is fixed bit for bit by this contract, for any view size and on every run:

    - d(p, q) = ((dx dx) + (dy dy)) + (dz dz) with dx = p.x - q.x, each step rounded to float32
      without fused multiply-adds; a distance counts only when it is finite;
    - the first point is the farthest from c, the float32 rounding of the float64 mean of the view's
      finite points (all three coordinates finite), summed in a fixed order; c = 0 without one;
    - after the first point s0 each point's key is d(p, s0), and after each later point s the key is
      min(key, d(p, s)); distances that do not count are skipped, so a point may have no key;
    - each round takes the untaken point with the largest key, ties to the lowest index, or, when no
      untaken point has a key, the lowest-index untaken point.

    So every row holds k distinct indices, a duplicate of a taken point (key 0) comes before any point
    with a NaN or inf coordinate, those come last in ascending index order, and
    ``farthest_point_sampling(x, k1)`` equals ``farthest_point_sampling(x, k2)[:, :k1]`` for k1 <= k2.

    Strided input is read in place (``pts[None]``, ``x[..., :3]``).  A view that fits on chip is
    sampled by one thread-block cluster, larger ones by one cooperative launch (csrc/pointcloud.cu); the
    call reads nothing back to the host and can be captured in a CUDA graph.

    Deliberate deviations from the reference:

    - the result is on the points' device, where the reference returns a CPU tensor;
    - equal keys resolve to the lowest index, where the reference's races leave the order unspecified;
    - points with a NaN or inf coordinate are taken in index order;
    - a finite point whose distance to the first point overflows to inf is not set aside for the rest
      of the call: a later finite distance gives it a key;
    - all views go through one call, where the reference loops over them;
    - errors raise ``ValueError`` (shape, k), ``TypeError`` (dtype) and ``NotImplementedError`` (CPU
      input), where the reference asserts.
    """
    func = "farthest_point_sampling"
    if points.ndim != 3 or points.shape[-1] != 3:
        raise ValueError(f"{func}: expected points of shape (batch_size, num_points, 3), got {tuple(points.shape)}")
    if not points.is_cuda:
        raise NotImplementedError(f"{func}: only CUDA is supported; points are on {points.device}")
    if points.dtype != torch.float32:
        raise TypeError(f"{func}: points should have dtype float32, got {points.dtype}")
    if isinstance(k, bool) or not isinstance(k, int):
        raise ValueError(f"{func}: k must be an int, got {type(k)}")
    B, N, _ = points.shape
    if not 0 <= k <= N:
        raise ValueError(f"{func}: k must satisfy 0 <= k <= num_points, but got k={k} and num_points={N}")
    dev = points.device
    nbytes, _, _ = _lib.farthest_point_sampling_workspace_bytes(B, N, k, dev, func)
    out = torch.empty((B, k), dtype=torch.int64, device=dev)
    if out.numel() == 0:
        return out
    _lib.call("dibr_b200_farthest_point_sampling", dev, B, N, k, points, *points.stride(), out,
              _lib.scratch(nbytes, dev), nbytes, what=func)
    return out
