"""TEST INFRASTRUCTURE — a torch restatement of the farthest-point-sampling contract of
kaolin_b200/csrc/pointcloud.cu, on either device.

Distances are separate elementwise float32 ops (no fused multiply-add), non-counting distances are
skipped with ``torch.where``, each round selects by ``argmax`` over the 64-bit candidate
(hi = 2 + key bits, 1 without a key, 0 when taken; lo = ~index), and the center is summed in float64
in the stated order: 1024-point chunks in index order, each reduced by the tree i + h for
h = 512, ..., 1, non-finite points contributing 0, the chunk sums added in index order.
"""
import torch

CHUNK = 1024


def center(points):
    """(B, N, 3) float32 -> (B, 3) float32: the float32 rounding of the float64 mean of each view's
    finite points in the contract's order, 0 for a view without one."""
    B, N, _ = points.shape
    finite = torch.isfinite(points).all(dim=-1, keepdim=True)
    p = torch.where(finite, points.double(), torch.zeros((), dtype=torch.float64, device=points.device))
    s = torch.cat([p, finite.double()], dim=-1)
    chunks = max(1, -(-N // CHUNK))
    s = torch.cat([s, s.new_zeros((B, chunks * CHUNK - N, 4))], dim=1).view(B, chunks, CHUNK, 4)
    h = CHUNK // 2
    while h >= 1:
        s = s[:, :, :h] + s[:, :, h:2 * h]
        h //= 2
    s = s[:, :, 0]
    total = s[:, 0]
    for c in range(1, chunks):
        total = total + s[:, c]
    n = total[:, 3:]
    return torch.where(n > 0, total[:, :3] / n, torch.zeros_like(total[:, :3])).float()


def distance(points, q):
    """d(p, q) = ((dx dx) + (dy dy)) + (dz dz) in float32, one rounding per op; q is (B, 1, 3)."""
    dx = points[..., 0] - q[..., 0]
    dy = points[..., 1] - q[..., 1]
    dz = points[..., 2] - q[..., 2]
    return (dx * dx + dy * dy) + dz * dz


def farthest_point_sampling(points, k):
    """(B, N, 3) float32 -> (B, k) int64 on the points' device, by the contract."""
    B, N, _ = points.shape
    dev = points.device
    out = torch.empty((B, k), dtype=torch.int64, device=dev)
    if B * k == 0:
        return out
    inf = torch.tensor(float("inf"), device=dev)
    lo = (2 ** 32 - 1) - torch.arange(N, device=dev, dtype=torch.int64)
    key = torch.full((B, N), float("inf"), device=dev)
    q = center(points)[:, None, :]
    for r in range(k):
        d = distance(points, q)
        counts = torch.isfinite(d)
        if r == 0:
            competing = torch.where(counts, d, inf)
        else:
            key = torch.where(counts, torch.minimum(key, d), key)
            competing = key
        bits = competing.contiguous().view(torch.int32).to(torch.int64)
        hi = torch.where(competing < 0, 0, torch.where(competing == inf, 1, 2 + bits))
        w = (hi * 2 ** 32 + lo).argmax(dim=1)
        out[:, r] = w
        key.scatter_(1, w[:, None], -1.0)
        q = points.gather(1, w[:, None, None].expand(B, 1, 3))
    return out
