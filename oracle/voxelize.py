"""TEST INFRASTRUCTURE — a torch restatement of the reference's voxelization (kaolin/ops/conversions/
trianglemesh.py:29-110, pointcloud.py:22-141, kaolin/ops/mesh/trianglemesh.py:340-458), with its
level-synchronous structure: a Python loop over views and, per view, one pass per subdivision level
that reads the number of split triangles back to the host and filters with a boolean mask.

Runs on the CPU and on CUDA.  It returns the sorted int64 (view, x, y, z) rows of every set voxel.
A point is kept when its rounded indices lie in [0, res-1], tested in floating point, so a NaN point
is dropped, as the reference drops it on the CPU and on CUDA.  Options:
  - ``prune``: skip triangles whose three vertices all quantise below 0 or all above res-1 on one
    axis (exact: no descendant could mark a voxel);
  - ``split_nonfinite``: False leaves triangles with a non-finite coordinate unsplit; True splits
    them as the reference does, which does not terminate when a coordinate is infinite.
"""
import torch


def normalize(points, origin=None, scale=None):
    if origin is None:
        origin = torch.min(points, dim=1)[0]
    if scale is None:
        scale = torch.max(torch.max(points, dim=1)[0] - origin, dim=1)[0]
    return (points - origin.unsqueeze(1)) / scale.view(-1, 1, 1)


def _quantize(p, res):
    """(N, 3) points -> (N, 3) int64 voxel indices of the points inside the grid."""
    q = torch.round(p * torch.tensor(res - 1, dtype=p.dtype, device=p.device))
    keep = ((q >= 0) & (q <= res - 1)).all(dim=1)
    return q[keep].long()


def _sq(a, b):
    d = a - b
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def _subdivision_midpoints(v, faces, res, prune, split_nonfinite, stats):
    """The midpoints the reference's subdivision adds for one view v (V, 3), level by level; adds the
    number of triangles tested to stats["nodes"]."""
    thr = torch.tensor(((res - 1) / (res ** 2)) ** 2, dtype=v.dtype).item()
    v1, v2, v3 = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    rm1 = torch.tensor(res - 1, dtype=v.dtype, device=v.device)
    out = []
    while True:
        stats["nodes"] = stats.get("nodes", 0) + v1.shape[0]
        m = torch.max(torch.stack([_sq(v1, v2), _sq(v2, v3), _sq(v3, v1)], dim=1), dim=1)[0]
        keep = m > thr
        if not split_nonfinite:
            keep &= torch.isfinite(torch.cat([v1, v2, v3], dim=1)).all(dim=1)
        if prune:
            q = torch.round(torch.stack([v1, v2, v3], dim=1) * rm1)        # (K, 3 vertices, 3 axes)
            out_lo = (q < 0).all(dim=1).any(dim=1)
            out_hi = (q > res - 1).all(dim=1).any(dim=1)
            keep &= ~(out_lo | out_hi)
        if int(torch.sum(keep)) == 0:
            break
        v1, v2, v3 = v1[keep], v2[keep], v3[keep]
        v4, v5, v6 = (v1 + v3) / 2, (v1 + v2) / 2, (v2 + v3) / 2
        out += [v4, v5, v6]
        v1, v2, v3 = torch.cat((v1, v2, v4, v3)), torch.cat((v4, v5, v5, v4)), torch.cat((v5, v6, v6, v6))
    return out


def voxel_rows(points, resolution, faces=None, prune=False, split_nonfinite=False, stats=None):
    """Normalised points (B, P, 3) and optional faces (F, 3) -> (nnz, 4) int64 sorted unique rows.
    ``stats`` (a dict) receives the number of triangles the subdivision tested, under "nodes"."""
    stats = {} if stats is None else stats
    rows = []
    for b in range(points.shape[0]):
        pts = [points[b]]
        if faces is not None and faces.shape[0]:
            pts += _subdivision_midpoints(points[b], faces.long(), resolution, prune, split_nonfinite, stats)
        q = _quantize(torch.cat(pts), resolution)
        rows.append(torch.cat([torch.full((q.shape[0], 1), b, dtype=torch.long, device=q.device), q], dim=1))
    if not rows:
        return torch.zeros((0, 4), dtype=torch.long, device=points.device)
    return torch.unique(torch.cat(rows), dim=0)


def dense(rows, batch, resolution, dtype):
    vg = torch.zeros((batch, resolution, resolution, resolution), dtype=dtype, device=rows.device)
    vg[rows[:, 0], rows[:, 1], rows[:, 2], rows[:, 3]] = 1
    return vg
