"""voxelgrids_to_cubic_meshes on sm_90a (csrc/cubic_meshes.cu) against the reference's own outputs
(tests/golden/cubic_meshes.npz) and the numpy restatement of the contract (oracle/cubic_meshes.py):
vertices and faces equal to both in both modes, every dtype and non-contiguous input, all views in one
call; box counts; the 0/255 winding; the documented edge cases and errors; one synchronising read per
call; byte-identical reruns; odd workspace addresses; 2 x 256^3 in bounded memory; the size limit."""
import warnings

import numpy as np
import pytest
import torch

from kaolin_b200 import _lib, synthetic
from kaolin_b200.ops import conversions
from kaolin_b200.ops.conversions import trianglemeshes_to_voxelgrids
from oracle import cubic_meshes as O
from test_cubic_meshes_cpu import MODES, SCENES, golden

pytestmark = pytest.mark.gpu
DEV = "cuda"
cubify = conversions.voxelgrids_to_cubic_meshes


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def check_against_oracle(grid, verts, faces, is_trimesh, what=""):
    """grid: the tensor the function was called with."""
    ref = grid.cpu()
    ref = ref.float() if ref.dtype in (torch.float16, torch.bfloat16) else ref
    ov, of = O.cubic_meshes(ref.numpy(), is_trimesh)
    assert len(verts) == len(faces) == grid.shape[0]
    for b in range(grid.shape[0]):
        assert verts[b].dtype == torch.float32 and faces[b].dtype == torch.int64
        assert verts[b].device == grid.device and faces[b].device == grid.device
        assert torch.equal(verts[b].cpu(), torch.from_numpy(ov[b])), (what, b)
        assert torch.equal(faces[b].cpu(), torch.from_numpy(of[b])), (what, b)


def dtypes_of(grid):
    """The stored dtype, float32, and for binary grids bool and uint8."""
    out = [grid.dtype.name, "float32"]
    if np.isin(grid, (0, 1)).all():
        out += ["bool", "uint8"]
    return sorted(set(out))


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", SCENES)
def test_equals_reference_golden(name, mode):
    grid, rv, rf = golden(name, mode)
    for dt in dtypes_of(grid):
        verts, faces = cubify(cuda(grid.astype(dt)), is_trimesh=MODES[mode])
        assert len(verts) == len(faces) == grid.shape[0]
        for b in range(grid.shape[0]):
            assert torch.equal(verts[b], cuda(rv[b])), (name, mode, dt, b)
            assert torch.equal(faces[b], cuda(rf[b])), (name, mode, dt, b)


RANDOM = {
    "d05_32": lambda r: r.random((2, 32, 32, 32)) < 0.05,
    "d50_40": lambda r: r.random((2, 40, 40, 40)) < 0.5,
    "d95_33": lambda r: r.random((1, 33, 33, 33)) < 0.95,
    "noncubic_37x64x50": lambda r: r.random((1, 37, 64, 50)) < 0.4,
    "thin_1x40x29": lambda r: r.random((2, 1, 40, 29)) < 0.5,
    "thin_23x1x1": lambda r: r.random((3, 23, 1, 1)) < 0.5,
    "thin_1x1x1": lambda r: r.random((3, 1, 1, 1)) < 0.5,
    # lattices of 31, 32, 33, 63, 64 and 65 points per row, and whole lattices of 32 k -+ 1
    "rows_30": lambda r: r.random((2, 3, 4, 30)) < 0.5,
    "rows_31": lambda r: r.random((2, 3, 4, 31)) < 0.5,
    "rows_32": lambda r: r.random((2, 3, 4, 32)) < 0.5,
    "rows_62_63_64": lambda r: r.random((2, 62, 63, 64)) < 0.5,
    "lattice_1x1x15": lambda r: r.random((3, 1, 1, 15)) < 0.5,     # 2 * 2 * 16 = 64 points
    "lattice_2x2x3": lambda r: r.random((3, 2, 2, 3)) < 0.5,       # 36 points
    "lattice_1x3x7": lambda r: r.random((3, 1, 3, 7)) < 0.5,       # 2 * 4 * 8 = 64 points
    "quarters": lambda r: (r.integers(0, 5, (2, 17, 19, 21)) / 4).astype(np.float32),
    "floats_any": lambda r: r.normal(0, 2, (2, 13, 11, 9)).astype(np.float32),
}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", list(RANDOM))
def test_equals_oracle_on_random_grids(name, mode):
    grid = RANDOM[name](np.random.default_rng(sum(map(ord, name))))
    g = cuda(grid)
    verts, faces = cubify(g, is_trimesh=MODES[mode])
    check_against_oracle(g, verts, faces, MODES[mode], name)


def test_batch_of_five_with_empty_views_interleaved():
    rng = np.random.default_rng(3)
    grid = rng.random((5, 19, 12, 17)) < 0.3
    grid[[0, 2, 4]] = False
    for tri in (True, False):
        g = cuda(grid)
        verts, faces = cubify(g, tri)
        check_against_oracle(g, verts, faces, tri)
        assert [len(v) for v in verts][::2] == [0, 0, 0] and all(len(f) for f in faces[1::2])


@pytest.mark.parametrize("dtype", [torch.bool, torch.uint8, torch.float32, torch.float64, torch.float16,
                                   torch.int32, torch.bfloat16])
def test_dtypes(dtype):
    rng = np.random.default_rng(4)
    base = torch.from_numpy(rng.integers(0, 2, (2, 21, 18, 13))).to(DEV)
    grid = (base > 0) if dtype == torch.bool else base.to(dtype)
    for tri in (True, False):
        verts, faces = cubify(grid, tri)
        check_against_oracle(grid, verts, faces, tri, str(dtype))
    if dtype in (torch.float64, torch.float16):       # fractional values, read as float32
        g = torch.from_numpy(rng.normal(0, 1.5, (2, 9, 10, 11))).to(DEV).to(dtype)
        verts, faces = cubify(g, False)
        check_against_oracle(g, verts, faces, False, str(dtype))


def test_non_contiguous_input():
    rng = np.random.default_rng(6)
    bits = cuda(rng.random((3, 20, 18, 24)) < 0.5)
    for big in (bits, bits.to(torch.uint8), bits.float()):
        for g in (big.permute(0, 3, 1, 2), big[:, ::2, 1:17, ::2], big.transpose(1, 3)[:, 2:]):
            assert not g.is_contiguous()
            for tri in (True, False):
                verts, faces = cubify(g, tri)
                check_against_oracle(g, verts, faces, tri)
                rv, rf = cubify(g.contiguous(), tri)
                assert all(torch.equal(a, b) for a, b in zip(verts + faces, rv + rf))


def test_voxelized_icospheres_at_128():
    v, f = synthetic.icosphere(5)
    rng = np.random.default_rng(7)
    views = np.stack([v * rng.uniform(0.6, 1.0) + rng.normal(scale=0.1, size=3) for _ in range(3)])
    g = trianglemeshes_to_voxelgrids(cuda(views.astype(np.float32)), cuda(f), 128)
    assert g.shape == (3, 128, 128, 128)
    for tri in (True, False):
        verts, faces = cubify(g, tri)
        check_against_oracle(g, verts, faces, tri)
        assert all(len(x) > 10000 for x in faces)


@pytest.mark.parametrize("shape", [(1, 1, 1), (3, 4, 5), (7, 2, 9), (31, 32, 33)])
def test_box_counts(shape):
    a, b, c = shape
    grid = torch.zeros((2, a + 3, b + 2, c + 4), dtype=torch.uint8, device=DEV)
    grid[0, 1:a + 1, 1:b + 1, 2:c + 2] = 1
    grid[1, :a, :b, :c] = 1
    verts, faces = cubify(grid, False)
    nq, nv = 2 * (a * b + b * c + c * a), (a + 1) * (b + 1) * (c + 1) - (a - 1) * (b - 1) * (c - 1)
    assert [f.shape for f in faces] == [(nq, 4)] * 2 and [v.shape for v in verts] == [(nv, 3)] * 2
    assert torch.equal(verts[1] + torch.tensor([1.0, 1.0, 2.0], device=DEV), verts[0])
    tv, tf = cubify(grid)
    assert [f.shape for f in tf] == [(2 * nq, 3)] * 2
    # every edge of the closed box is shared by exactly two triangles, in opposite directions
    e = torch.cat([tf[0][:, [0, 1]], tf[0][:, [1, 2]], tf[0][:, [2, 0]]])
    assert torch.unique(e, dim=0).shape[0] == e.shape[0]
    assert torch.equal(torch.unique(e, dim=0), torch.unique(e.flip(1), dim=0))


def test_0_255_winds_like_0_1():
    rng = np.random.default_rng(8)
    ones = cuda((rng.random((2, 23, 17, 19)) < 0.5).astype(np.uint8))
    for tri in (True, False):
        a = cubify(ones, tri)
        b = cubify(ones * 255, tri)
        c = cubify(ones.float() * 3.0, tri)
        assert all(torch.equal(x, y) and torch.equal(x, z) for x, y, z in zip(a[0] + a[1], b[0] + b[1], c[0] + c[1]))


def test_empty_batch_zero_sizes_and_errors():
    for tri, k in ((True, 3), (False, 4)):
        for grid in (torch.zeros((3, 5, 6, 7), device=DEV), torch.full((2, 4, 4, 4), 0.4, device=DEV)):
            verts, faces = cubify(grid, tri)
            assert len(verts) == len(faces) == grid.shape[0]
            assert all(v.shape == (0, 3) and v.dtype == torch.float32 and v.is_cuda for v in verts)
            assert all(f.shape == (0, k) and f.dtype == torch.int64 and f.is_cuda for f in faces)
        assert cubify(torch.zeros((0, 3, 3, 3), device=DEV), tri) == ([], [])
        verts, faces = cubify(torch.ones((2, 3, 0, 3), device=DEV), tri)
        assert [v.shape for v in verts] == [(0, 3)] * 2 and [f.shape for f in faces] == [(0, k)] * 2
    with pytest.raises(NotImplementedError):
        cubify(torch.ones((1, 2, 2, 2)))
    with pytest.raises(ValueError):
        cubify(torch.ones((2, 2, 2), device=DEV))
    with pytest.raises(ValueError):
        cubify(torch.ones((1, 1, 2, 2, 2), device=DEV))


def test_one_sync_per_call():
    rng = np.random.default_rng(9)
    grid = cuda(rng.random((3, 24, 20, 22)) < 0.4)
    cubify(grid)
    torch.cuda.synchronize()
    for tri in (True, False):
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                cubify(grid, tri)
            finally:
                torch.cuda.set_sync_debug_mode("default")
        syncs = [w for w in caught if "called a synchronizing" in str(w.message)]
        assert len(syncs) == 1, [str(w.message) for w in caught]


def test_reruns_are_byte_identical():
    rng = np.random.default_rng(10)
    grid = cuda(rng.random((2, 48, 40, 44)) < 0.5)
    runs = []
    for _ in range(3):
        verts, faces = cubify(grid)
        runs.append((torch.cat(verts).cpu().numpy().tobytes(), torch.cat(faces).cpu().numpy().tobytes()))
    assert runs[0] == runs[1] == runs[2]


def test_workspace_at_an_odd_address(monkeypatch):
    rng = np.random.default_rng(11)
    grid = cuda(rng.random((2, 24, 25, 26)) < 0.5)
    want = [torch.cat(x) for x in cubify(grid)]
    scratch, odd = _lib.scratch, []
    monkeypatch.setattr(_lib, "scratch", lambda n, device: odd.append(n) or scratch(int(n) + 1, device)[1:])
    got = [torch.cat(x) for x in cubify(grid)]
    assert odd
    assert all(torch.equal(a, b) for a, b in zip(want, got))


def test_256_cubed_two_views_in_bounded_memory():
    n, B = 256, 2
    c = torch.arange(n, device=DEV, dtype=torch.float32) - n / 2 + 0.5
    r2 = c[:, None, None] ** 2 + c[None, :, None] ** 2 + c[None, None, :] ** 2
    grid = torch.stack([r2 < (0.4 * n) ** 2, (r2 < (0.45 * n) ** 2) & (r2 > (0.3 * n) ** 2)]).to(torch.uint8)
    del c, r2
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    verts, faces = cubify(grid)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    out = sum(v.numel() * 4 + f.numel() * 8 for v, f in zip(verts, faces))
    bound = _lib.cubic_meshes_workspace_bytes(B, n, n, n, "q") + out + 32 * 1024 * 1024
    assert peak <= bound, (peak, bound)
    for b in range(B):
        v1, f1 = cubify(grid[b:b + 1])
        assert torch.equal(verts[b], v1[0]) and torch.equal(faces[b], f1[0])
        assert int(faces[b].min()) == 0 and int(faces[b].max()) == verts[b].shape[0] - 1


def test_size_limit_raises_without_allocating():
    one = torch.ones((1, 1, 1, 1), dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    for shape in ((1, 812, 812, 812), (32, 255, 255, 255), (1, 2 ** 16, 2 ** 15, 1)):
        with pytest.raises(RuntimeError, match="voxelgrids_to_cubic_meshes"):
            cubify(one.expand(*shape))
    assert torch.cuda.memory_allocated() == before
    v, f = cubify(one.expand(1, 40, 50, 60), False)          # stride 0 is read in place
    assert f[0].shape == (2 * (40 * 50 + 50 * 60 + 60 * 40), 4)
