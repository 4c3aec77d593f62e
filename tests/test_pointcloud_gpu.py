"""kaolin.ops.pointcloud on the GPU: farthest_point_sampling bit-equal to the contract's torch oracle
(oracle/pointcloud.py, run on CUDA) on random, tied, duplicated, non-finite, overflowing and subnormal
clouds, at every cluster-size boundary and on both sides of the cluster-to-grid boundary, with the
farthest-point property checked in float64 on every scene it covers; the prefix property, reruns, the
result's device, host reads, CUDA-graph capture, peak memory and the errors; center_points bit-equal to
the reference's outputs in tests/golden/pointcloud.npz."""
import numpy as np
import pytest
import torch

from kaolin_b200 import _lib
from kaolin_b200.ops import pointcloud as pc
from oracle import pointcloud as opc
from test_pointcloud_cpu import CENTER, check_farthest

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def plan(B, N, k):
    return _lib.farthest_point_sampling_workspace_bytes(B, N, k, DEV, "plan")


def run(points, k, prop=True):
    """The kernel's indices, asserted equal to the oracle's (and to the farthest-point property)."""
    got = pc.farthest_point_sampling(points, k)
    assert got.dtype == torch.int64 and got.device == points.device and got.shape == (points.shape[0], k)
    want = opc.farthest_point_sampling(points, k)
    assert torch.equal(got, want), (got != want).nonzero()[:5].tolist()
    if prop:
        check_farthest(points, got)
    return got


def scene_uniform():
    return torch.rand((3, 5000, 3), device=DEV, generator=gen(1)), 500


def scene_blobs():
    g = gen(2)
    centers = torch.randint(-5, 5, (2, 4000, 3), device=DEV, generator=g).float()
    return centers + 0.01 * torch.randn((2, 4000, 3), device=DEV, generator=g), 400


def scene_lattice():
    a = torch.arange(16.0, device=DEV)
    return torch.stack(torch.meshgrid(a, a, a, indexing="ij"), -1).reshape(1, -1, 3), 4096


def scene_half_identical():
    p = torch.rand((2, 3000, 3), device=DEV, generator=gen(3))
    p[:, 1500:] = p[:, :1]
    return p, 1700


def scene_all_identical():
    return torch.full((2, 700, 3), 0.25, device=DEV), 700


def scene_nonfinite_not_taken():
    p = torch.randn((2, 3000, 3), device=DEV, generator=gen(4))
    p[0, ::13, 0] = float("nan")
    p[1, 5:40, 2] = float("inf")
    p[1, 100] = -float("inf")
    return p, 200


def scene_nonfinite_taken():
    p = torch.randn((2, 900, 3), device=DEV, generator=gen(5))
    p[0, ::9, 1] = float("nan")
    p[1, 3::11] = float("inf")
    p[1, 0] = float("nan")
    return p, 900


def scene_single_nan_coordinate():
    p = torch.rand((1, 2000, 3), device=DEV, generator=gen(6))
    p[0, 777, 2] = float("nan")
    return p, 2000


def scene_subnormal_and_signed_zero():
    g = gen(7)
    p = torch.rand((2, 1500, 3), device=DEV, generator=g)
    p[0, :500] = torch.rand((500, 3), device=DEV, generator=g) * 1e-40
    p[0, 500:600] = -0.0
    p[0, 600:700] = 0.0
    p[1] = torch.rand((1500, 3), device=DEV, generator=g) * 1e-41 * torch.where(
        torch.rand((1500, 3), device=DEV, generator=g) < 0.5, -1.0, 1.0)
    return p, 1500


SCENES = {f.__name__[6:]: f for f in (scene_uniform, scene_blobs, scene_lattice, scene_half_identical,
                                      scene_all_identical, scene_nonfinite_not_taken, scene_nonfinite_taken,
                                      scene_single_nan_coordinate, scene_subnormal_and_signed_zero)}


@pytest.mark.parametrize("name", sorted(SCENES))
def test_scene_equals_oracle_and_is_farthest(name):
    points, k = SCENES[name]()
    run(points, k)


def test_distance_overflow_equals_oracle():
    """Coordinates near 1e19-1e20: float32 squared distances overflow to inf and do not count, so such
    points compete without a key until a finite distance gives them one (the float64 property does
    not hold by design here)."""
    g = gen(8)
    p = torch.rand((2, 3000, 3), device=DEV, generator=g)
    p[0, ::3] *= 1e20
    p[1, :10] = torch.rand((10, 3), device=DEV, generator=g) * 1e20 + 1e19
    got = run(p, 3000, prop=False)
    assert all(len(set(r)) == 3000 for r in got.tolist())
    # a far point whose distance to the first point overflows is still taken by its later finite key
    q = torch.tensor([[[0.0, 0, 0], [1e19, 0, 0], [2e19, 0, 0], [3e19, 1, 0], [0.5, 0.5, 0]]], device=DEV)
    run(q, 5, prop=False)


@pytest.mark.parametrize("B,N,k", [(1, 1, 1), (1, 1, 0), (2, 7, 0), (0, 5, 3), (0, 0, 0), (3, 9, 9), (1, 40, 1)])
def test_small_and_empty_shapes(B, N, k):
    points = torch.randn((B, N, 3), device=DEV, generator=gen(9))
    got = run(points, k)
    if B and k:
        assert got.shape == (B, k)


def test_batch_of_64_views():
    points = torch.randn((64, 2000, 3), device=DEV, generator=gen(10)) * torch.arange(1, 65, device=DEV)[:, None, None]
    got = run(points, 64)
    for b in (0, 17, 63):
        assert torch.equal(got[b:b + 1], pc.farthest_point_sampling(points[b:b + 1], 64))


def test_strided_input_is_read_in_place():
    g = gen(11)
    x = torch.randn((3, 4000, 6), device=DEV, generator=g)
    want = pc.farthest_point_sampling(x[..., :3].contiguous(), 300)
    assert torch.equal(pc.farthest_point_sampling(x[..., :3], 300), want)
    assert torch.equal(want, opc.farthest_point_sampling(x[..., :3], 300))
    y = x[..., :3].permute(0, 2, 1).contiguous().permute(0, 2, 1)
    assert torch.equal(pc.farthest_point_sampling(y, 300), want)
    single = x[1, :, :3]
    assert torch.equal(pc.farthest_point_sampling(single[None], 300), want[1:2])


def boundaries():
    """Every N where the plan changes its path or cluster size (found by asking the workspace query),
    with N on both sides."""
    def state(N):
        _, path, cluster = plan(1, N, 1)
        return path, cluster

    def first_with(pred, lo, hi):
        while lo < hi:
            mid = (lo + hi) // 2
            if pred(mid):
                hi = mid
            else:
                lo = mid + 1
        return lo

    top = 1 << 22
    out, N = [], 1
    while True:
        s = state(N)
        if s[0] == _lib.FPS_GRID:
            break
        nxt = first_with(lambda n: state(n) != s, N, top)
        out.append((nxt - 1, state(nxt - 1), nxt, state(nxt)))
        N = nxt
    return out


def test_plan_boundaries_cover_every_cluster_size_and_the_grid():
    b = boundaries()
    sizes = [lo[1] for _, lo, _, _ in b] + [b[-1][3][1]]
    assert b[-1][3][0] == _lib.FPS_GRID and b[-1][1][0] == _lib.FPS_CLUSTER
    assert sizes[:-1] == list(range(1, len(sizes)))      # 1, 2, ..., the largest cluster
    assert len(sizes) - 1 in (8, 16)


def test_every_boundary_equals_oracle():
    """N on both sides of every cluster-size boundary and of the cluster-to-grid boundary."""
    seen = set()
    for seed, (n_lo, s_lo, n_hi, s_hi) in enumerate(boundaries()):
        for N, s in ((n_lo, s_lo), (n_hi, s_hi)):
            points = torch.randn((1, N, 3), device=DEV, generator=gen(100 + seed)) * 3
            points[0, N // 2] = float("nan")
            got = run(points, 48, prop=False)
            check_farthest(points, got)
            seen.add(s)
    assert any(p == _lib.FPS_GRID for p, _ in seen)


def test_shared_memory_tier_and_grid_path_views():
    """A view that needs the cluster's shared memory, and grid-path views with B > 1 (points in the
    workspace past each CTA's on-chip share)."""
    b = boundaries()
    regs, largest, grid_n = b[0][0], b[-1][1][1], b[-1][2]
    for N in (largest * regs, largest * regs + 1, grid_n - 1000):    # registers only, then shared memory
        assert plan(1, N, 8)[1:] == (_lib.FPS_CLUSTER, largest)
        run(torch.rand((2, N, 3), device=DEV, generator=gen(N)), 200, prop=False)
    assert plan(3, grid_n + 5, 8)[1] == _lib.FPS_GRID
    run(torch.randn((3, grid_n + 5, 3), device=DEV, generator=gen(13)), 100, prop=False)


def test_prefix_property_and_byte_identical_reruns():
    for N in (5000, 200000):
        points = torch.randn((2, N, 3), device=DEV, generator=gen(14))
        full = pc.farthest_point_sampling(points, 700)
        for k1 in (0, 1, 2, 255, 256, 257, 699):
            assert torch.equal(pc.farthest_point_sampling(points, k1), full[:, :k1])
        for _ in range(3):
            assert torch.equal(pc.farthest_point_sampling(points, 700), full)


def test_no_host_synchronisation():
    small = torch.randn((4, 3000, 3), device=DEV, generator=gen(15))
    big = torch.randn((1, 400000, 3), device=DEV, generator=gen(16))
    want = [pc.farthest_point_sampling(small, 100), pc.farthest_point_sampling(big, 50)]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = [pc.farthest_point_sampling(small, 100), pc.farthest_point_sampling(big, 50)]
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert all(torch.equal(a, b) for a, b in zip(got, want))


@pytest.mark.parametrize("N", [3000, 400000])
def test_cuda_graph_capture_and_replay(N):
    points = torch.randn((2, N, 3), device=DEV, generator=gen(17))
    eager = pc.farthest_point_sampling(points, 300)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        pc.farthest_point_sampling(points, 300)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = pc.farthest_point_sampling(points, 300)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    points.copy_(torch.randn((2, N, 3), device=DEV, generator=gen(18)))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, pc.farthest_point_sampling(points, 300))


@pytest.mark.parametrize("B,N,k", [(1, 10 ** 6, 10 ** 4), (1, 1 << 22, 1024), (32, 8192, 1024)])
def test_large_runs_equal_oracle(B, N, k):
    points = torch.randn((B, N, 3), device=DEV, generator=gen(19)) * torch.tensor([1.0, 2.0, 0.5], device=DEV)
    got = pc.farthest_point_sampling(points, k)
    assert torch.equal(got, opc.farthest_point_sampling(points, k))
    if B > 1:    # the float64 check of 10^4 rounds over 10^6 points would take minutes on the host
        check_farthest(points[:2], got[:2])


@pytest.mark.parametrize("B,N,k", [(1, 1 << 22, 256), (32, 8192, 1024), (2, 100000, 512)])
def test_peak_memory_is_the_output_and_the_layout(B, N, k):
    points = torch.randn((B, N, 3), device=DEV, generator=gen(20))
    nbytes = plan(B, N, k)[0]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = pc.farthest_point_sampling(points, k)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak <= B * k * 8 + nbytes + 2 * 512, (peak, B * k * 8 + nbytes)
    del out


def test_errors():
    p = torch.randn((2, 10, 3), device=DEV)
    with pytest.raises(TypeError):
        pc.farthest_point_sampling(p.double(), 2)
    with pytest.raises(TypeError):
        pc.farthest_point_sampling(p.half(), 2)
    for k in (-1, 11):
        with pytest.raises(ValueError):
            pc.farthest_point_sampling(p, k)
    with pytest.raises(ValueError):
        pc.farthest_point_sampling(p[..., :2], 2)
    with pytest.raises(ValueError):
        pc.center_points(p[0])


@pytest.mark.parametrize("name", sorted(CENTER))
def test_center_points_equals_reference_golden(name):
    sc = CENTER[name]
    pts = torch.from_numpy(sc["points"]).to(DEV)
    plain = pc.center_points(pts)
    assert plain.dtype == pts.dtype and plain.device == pts.device
    np.testing.assert_array_equal(plain.cpu().numpy(), sc["plain"])
    norm = pc.center_points(pts, normalize=True, eps=float(sc["eps"]))
    np.testing.assert_array_equal(norm.cpu().numpy(), sc["normalized"])
