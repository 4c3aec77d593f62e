"""kaolin.ops.pointcloud without a GPU: the torch oracle (oracle/pointcloud.py) against the farthest-point
property and a direct restatement of the center's summation order, center_points' CPU refusal and
argument errors, the plan and workspace layout of op_layouts.h, and the C ABI's host-side errors.

``check_farthest`` is shared with tests/test_pointcloud_gpu.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from kaolin_b200 import _lib
from kaolin_b200.ops import pointcloud as pc
from oracle import pointcloud as opc

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "pointcloud.npz")
SRC = os.path.join(ROOT, "tests", "host_math", "pointcloud_layout.cpp")
HDR = os.path.join(ROOT, "kaolin_b200", "csrc", "op_layouts.h")
LIB = os.path.join(ROOT, "tests", "host_math", "_build", "pointcloud_layout.so")
ALIGN = 256
INT32_MAX = 2 ** 31 - 1

_G = np.load(GOLDEN)
CENTER = {}
for _k in _G.files:
    _f, _name, _item = _k.split("__")
    CENTER.setdefault(_name, {})[_item] = _G[_k]


def check_farthest(points, idx, rtol=1e-5):
    """The farthest-point property in float64, written from its statement: every row holds distinct
    indices; the first is (within a tolerance) the farthest finite point from the mean of the view's
    finite points; each later one is the farthest untaken finite point from the taken finite set; once
    the finite points are used up, the rest are the non-finite points in ascending index order.
    Points whose float32 squared distances can overflow are outside this statement."""
    p = points.detach().double().cpu()
    idx = idx.cpu()
    B, N, _ = p.shape
    k = idx.shape[1]
    for b in range(B):
        row = idx[b].tolist()
        assert len(set(row)) == k and all(0 <= i < N for i in row), b
        fin = torch.isfinite(p[b]).all(-1)
        if not fin.any():
            assert row == list(range(k)), b
            continue
        x = torch.where(fin[:, None], p[b], torch.zeros(()))
        mean = x[fin].mean(0)
        scale2 = float(((x[fin] - mean) ** 2).sum(-1).max())
        atol = 1e-6 * scale2 + 2.0 ** -120

        def dist(q):
            return torch.where(fin, ((x - q) ** 2).sum(-1), torch.tensor(-1.0, dtype=torch.float64))

        d = dist(mean)
        taken = torch.zeros(N, dtype=torch.bool)
        mind = None
        nonfinite = [i for i in range(N) if not fin[i]]
        for r, s in enumerate(row):
            left = fin & ~taken
            if not left.any():
                assert row[r:] == [i for i in nonfinite if not taken[i]][:k - r], (b, r)
                break
            assert fin[s], (b, r, s)
            best = float(d[left].max()) if mind is None else float(mind[left].max())
            got = float(d[s]) if mind is None else float(mind[s])
            assert got >= best * (1 - rtol) - atol, (b, r, s, got, best)
            taken[s] = True
            ds = dist(x[s])
            mind = ds if mind is None else torch.minimum(mind, ds)


def clouds():
    g = torch.Generator().manual_seed(3)
    yield "uniform", torch.rand((2, 700, 3), generator=g), 64
    yield "blobs", torch.randn((1, 900, 3), generator=g) * 0.05 + torch.randint(0, 4, (1, 900, 1), generator=g), 100
    lattice = torch.stack(torch.meshgrid(*[torch.arange(6.0)] * 3, indexing="ij"), -1).reshape(1, -1, 3)
    yield "lattice", lattice, 216
    dup = torch.rand((1, 300, 3), generator=g)
    dup[0, 150:] = dup[0, 0]
    yield "half_duplicate", dup, 200
    bad = torch.rand((1, 200, 3), generator=g)
    bad[0, [3, 50, 199], 1] = float("nan")
    bad[0, [7, 8], 0] = float("inf")
    yield "nonfinite_taken", bad, 200
    yield "all_same", torch.ones((1, 50, 3)), 50


@pytest.mark.parametrize("name,points,k", list(clouds()), ids=[c[0] for c in clouds()])
def test_oracle_satisfies_the_farthest_point_property(name, points, k):
    idx = opc.farthest_point_sampling(points, k)
    check_farthest(points, idx)
    assert torch.equal(opc.farthest_point_sampling(points, k // 2), idx[:, :k // 2])


def test_oracle_ties_go_to_the_lowest_index_and_nonfinite_points_come_last():
    pts = torch.tensor([[[0.0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 0],
                         [float("nan"), 0, 0], [1, 0, 0]]])
    idx = opc.farthest_point_sampling(pts, 8)[0].tolist()
    # center (0.125, 0, 0): -1 is farthest; then 1 (d 4), its duplicate 7 only after every keyed point
    assert idx[:2] == [2, 1]
    assert idx[-1] == 6 and idx.index(7) > idx.index(3) and idx.index(7) > idx.index(4)


def test_center_order_is_restated_exactly():
    """The oracle's center against a scalar float64 loop in the stated order, for N across chunk
    borders and with non-finite points."""
    g = torch.Generator().manual_seed(5)
    for N in (1, 5, 1023, 1024, 1025, 3000):
        pts = torch.randn((2, N, 3), generator=g) * 1e3 + 7
        pts[1, ::7, 2] = float("nan")
        for b in range(2):
            x = pts[b].double().numpy()
            fin = np.isfinite(x).all(-1)
            S = None
            for c0 in range(0, N, 1024):
                s = np.zeros((1024, 4))
                n = min(1024, N - c0)
                s[:n, :3] = np.where(fin[c0:c0 + n, None], x[c0:c0 + n], 0.0)
                s[:n, 3] = fin[c0:c0 + n]
                h = 512
                while h >= 1:
                    s = s[:h] + s[h:2 * h]
                    h //= 2
                S = s[0] if S is None else S + s[0]
            want = (S[:3] / S[3]).astype(np.float32) if S[3] > 0 else np.zeros(3, np.float32)
            assert np.array_equal(opc.center(pts)[b].numpy(), want), (N, b)
    assert torch.equal(opc.center(torch.full((1, 4, 3), float("nan"))), torch.zeros((1, 3)))


@pytest.mark.parametrize("name", sorted(CENTER))
def test_center_points_expression_matches_the_golden_on_cpu(name):
    """The expression of center_points (its body without the device check) equals the reference's
    outputs; the GPU tests hold the public function to the same goldens on CUDA."""
    sc = CENTER[name]
    pts = torch.from_numpy(sc["points"])
    lo, hi = torch.aminmax(pts, dim=1, keepdim=True)
    out = pts - (lo + hi) / 2
    np.testing.assert_array_equal(out.numpy(), sc["plain"])
    norm = out / (hi - lo).amax(dim=-1, keepdim=True).clamp(min=float(sc["eps"]))
    np.testing.assert_array_equal(norm.numpy(), sc["normalized"])


def test_golden_covers_every_dtype_and_nan():
    assert {n.rsplit("_", 1)[1] for n in CENTER} == {"float16", "float32", "float64"}
    assert any(np.isnan(CENTER[n]["plain"]).any() for n in CENTER)


def test_cpu_input_and_argument_errors():
    with pytest.raises(NotImplementedError):
        pc.center_points(torch.zeros((1, 4, 3)))
    with pytest.raises(NotImplementedError):
        pc.farthest_point_sampling(torch.zeros((1, 4, 3)), 2)
    for bad in (torch.zeros((4, 3)), torch.zeros((1, 4, 2)), torch.zeros((1, 1, 4, 3))):
        with pytest.raises(ValueError):
            pc.farthest_point_sampling(bad, 1)


# ---------------------------------------------------------------------------------------------
# Plan, layout and the C ABI's host-side checks.

@pytest.fixture(scope="module")
def lay():
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(SRC), os.path.getmtime(HDR)):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", LIB, SRC])
    lib = ctypes.CDLL(LIB)
    lib.fps_layout_of.argtypes = [ctypes.c_int64] * 3 + [ctypes.c_int, ctypes.POINTER(ctypes.c_int64)]
    lib.fps_constants.argtypes = [ctypes.POINTER(ctypes.c_int64)]
    lib.fps_carve.argtypes = [ctypes.c_uint64] * 3
    lib.fps_carve.restype = ctypes.c_int64
    return lib


def layout(lay, B, N, k, max_cluster):
    out = (ctypes.c_int64 * 12)()
    lay.fps_layout_of(B, N, k, max_cluster, out)
    path, cluster, smem, total = out[:4]
    pieces = [(out[4 + 2 * i], out[5 + 2 * i]) for i in range(4)]
    return path, cluster, smem, total, pieces


def constants(lay):
    out = (ctypes.c_int64 * 4)()
    lay.fps_constants(out)
    return tuple(out)


def test_plan_capacity_boundaries(lay):
    T, R, S, chunk = constants(lay)
    regs, onchip = T * R, T * (R + S)
    assert chunk == 1024 and T * S * 16 <= 227 * 1024     # a CTA's shared-memory points fit on one SM
    for maxc in (16, 8, 1):
        for c in range(1, maxc + 1):
            assert layout(lay, 1, c * regs, 1, maxc)[:3] == (_lib.FPS_CLUSTER, c, 0)
            if c < maxc:
                assert layout(lay, 1, c * regs + 1, 1, maxc)[:3] == (_lib.FPS_CLUSTER, c + 1, 0)
        path, cluster, smem = layout(lay, 1, maxc * regs + 1, 1, maxc)[:3]
        assert (path, cluster, smem) == (_lib.FPS_CLUSTER, maxc, 1)
        assert layout(lay, 1, maxc * onchip, 1, maxc)[:3] == (_lib.FPS_CLUSTER, maxc, S)
        assert layout(lay, 1, maxc * onchip + 1, 1, maxc)[0] == _lib.FPS_GRID
    assert layout(lay, 0, 100, 1, 16)[0] == 0 and layout(lay, 3, 100, 0, 16)[0] == 0


@pytest.mark.parametrize("B,N,k", [(1, 1, 1), (4, 5000, 100), (32, 8192, 1024), (1, 10 ** 5, 1024),
                                   (1, 10 ** 6, 10 ** 4), (1, 2 ** 22, 1024), (64, 327681, 3)])
def test_layout_pieces_alignment_and_carve(lay, B, N, k):
    path, _, _, total, pieces = layout(lay, B, N, k, 16)
    chunks = -(-N // 1024)
    grid = path == _lib.FPS_GRID
    assert [p[1] for p in pieces] == [B * chunks * 32, B * 16, grid * B * 24, grid * B * N * 16]
    end = 0
    for at, n in pieces:
        assert at % ALIGN == 0 and at >= end
        end = at + n
    assert total == end + ALIGN
    for offset in (0, 1, 3, 8, 255):
        ws = 0x10000 + offset
        origin = lay.fps_carve(ws, total, total)
        assert 0 <= origin < ALIGN and (ws + origin) % ALIGN == 0
        assert all(origin + at + n <= total for at, n in pieces)
        assert lay.fps_carve(ws, total - 1, total) == -1


def test_c_abi_host_side_errors():
    lib = _lib.lib()
    n, path, cluster = ctypes.c_size_t(0), ctypes.c_int(0), ctypes.c_int(0)
    q = lib.dibr_b200_farthest_point_sampling_workspace_bytes
    r = (ctypes.byref(n), ctypes.byref(path), ctypes.byref(cluster))
    assert q(1, INT32_MAX, 1, *r) == _lib.ESIZE
    assert q(1, INT32_MAX - 1, INT32_MAX, *r) == _lib.EINVAL     # k > N
    assert q(-1, 4, 1, *r) == _lib.EINVAL
    assert q(1, -4, 1, *r) == _lib.EINVAL
    assert q(1, 4, -1, *r) == _lib.EINVAL
    assert q(1, 4, 5, *r) == _lib.EINVAL
    assert q(1, 4, 1, None, ctypes.byref(path), ctypes.byref(cluster)) == _lib.EINVAL
    assert q(0, 4, 2, *r) == 0 and path.value == 0                 # nothing to do: no device query
    assert q(3, 4, 0, *r) == 0 and path.value == 0
    fps = lib.dibr_b200_farthest_point_sampling
    assert fps(1, INT32_MAX, 1, 4096, 3 * 4, 3, 1, 4096, 4096, 1 << 20, None) == _lib.ESIZE
    assert fps(1, 4, 5, 4096, 12, 3, 1, 4096, 4096, 1 << 20, None) == _lib.EINVAL
    assert fps(1, 4, 2, None, 12, 3, 1, 4096, 4096, 1 << 20, None) == _lib.EINVAL
    assert fps(1, 4, 2, 4096, 12, 3, 1, None, 4096, 1 << 20, None) == _lib.EINVAL
    assert fps(0, 4, 2, None, 12, 3, 1, None, None, 0, None) == 0        # nothing to do
    assert fps(2, 4, 0, None, 12, 3, 1, None, None, 0, None) == 0
    with pytest.raises(RuntimeError):
        _lib.farthest_point_sampling_workspace_bytes(1, INT32_MAX, 1, None, "fps")
