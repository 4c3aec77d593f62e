"""trianglemeshes_to_voxelgrids and pointclouds_to_voxelgrids on the GPU: bit-equal to the reference's
outputs in tests/golden/voxelize.npz, dense and sparse; equal to the torch oracle (oracle/voxelize.py)
run on CUDA on seeded scenes at full size; the documented deviations, errors and limits; host reads,
reruns, workspace alignment and peak memory."""
import ctypes
import warnings

import numpy as np
import pytest
import torch

from kaolin_b200 import _lib, synthetic
from kaolin_b200.ops.conversions import pointclouds_to_voxelgrids, trianglemeshes_to_voxelgrids
from oracle import voxelize as ov
from test_voxelize_cpu import SCENES, as_torch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
CUBE_V = [[x, y, z] for x in (0., 1.) for y in (0., 1.) for z in (0., 1.)]
CUBE_F = [[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1],
          [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]]


def run(sc, sparse, device=DEV):
    v, f, o, s = as_torch(sc, device)
    if sc["kind"] == "mesh":
        return trianglemeshes_to_voxelgrids(v, f, sc["res"], o, s, return_sparse=sparse)
    return pointclouds_to_voxelgrids(v, sc["res"], o, s, return_sparse=sparse)


def rows_of(dense):
    return torch.nonzero(dense).T


@pytest.mark.parametrize("name", sorted(SCENES))
def test_dense_equals_reference_golden(name):
    sc = SCENES[name]
    out = run(sc, False)
    assert out.dtype == sc["dtype"] and tuple(out.shape) == sc["shape"]
    ref = torch.zeros(sc["shape"], dtype=sc["dtype"])
    ref[tuple(torch.from_numpy(sc["rows"]))] = 1
    assert torch.equal(out.cpu(), ref)


@pytest.mark.parametrize("name", sorted(SCENES))
def test_sparse_equals_reference_golden(name):
    sc = SCENES[name]
    out = run(sc, True)
    assert out.layout == torch.sparse_coo and out.dtype == sc["dtype"] and tuple(out.shape) == sc["shape"]
    assert out.is_coalesced() == sc["coalesced"]
    np.testing.assert_array_equal(out._indices().cpu().numpy(), sc["rows"])
    assert torch.equal(out._values().cpu(), torch.ones(sc["rows"].shape[1], dtype=sc["dtype"]))


def check_against_oracle(v, f, res, origin=None, scale=None, dense=True):
    p = ov.normalize(v, origin, scale)
    rows = ov.voxel_rows(p, res, f, prune=True)
    if f is None:
        call = lambda sparse: pointclouds_to_voxelgrids(v, res, origin, scale, return_sparse=sparse)
    else:
        call = lambda sparse: trianglemeshes_to_voxelgrids(v, f, res, origin, scale, return_sparse=sparse)
    assert torch.equal(call(True)._indices(), rows.T)
    if dense:
        assert torch.equal(rows_of(call(False)), rows.T)
    return rows


def soup(B, F, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    v = torch.rand((B, 3 * F, 3), generator=g, dtype=torch.float64)
    v[:, 1::3] = v[:, 0::3] + 0.2 * (torch.rand((B, F, 3), generator=g, dtype=torch.float64) - 0.5)
    v[:, 2::3] = v[:, 0::3] + 0.2 * (torch.rand((B, F, 3), generator=g, dtype=torch.float64) - 0.5)
    return v.to(dtype).to(DEV), torch.arange(3 * F, device=DEV).view(F, 3)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("res", [17, 128])
def test_triangle_soups_equal_the_oracle(dtype, res):
    v, f = soup(3, 500, seed=res, dtype=dtype)
    check_against_oracle(v, f, res)


def test_icosphere_level5_four_views_at_256_equal_the_oracle():
    v0, f = synthetic.icosphere(5)
    rng = np.random.default_rng(3)
    v = np.stack([v0 * (1 + 0.05 * rng.uniform(-1, 1, (v0.shape[0], 1))) for _ in range(4)]).astype(np.float32)
    check_against_oracle(torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV), 256)


def test_zoomed_view_at_512_equals_the_oracle():
    v0, f = synthetic.icosphere(3)
    v = torch.from_numpy(v0[None].astype(np.float32)).to(DEV)
    f = torch.from_numpy(f).to(DEV)
    origin = torch.tensor([[0.7, -0.2, -0.2]], device=DEV)
    scale = torch.tensor([0.4], device=DEV)
    rows = check_against_oracle(v, f, 512, origin, scale)
    assert rows.shape[0] > 1000


def test_million_point_clouds_equal_the_oracle():
    g = torch.Generator(device=DEV).manual_seed(5)
    p = torch.randn((4, 10 ** 6, 3), generator=g, device=DEV)
    check_against_oracle(p, None, 256)
    check_against_oracle(p.double(), None, 64)


def test_infinite_faces_are_not_split_and_nan_points_are_dropped():
    v = torch.tensor(CUBE_V).repeat(2, 1)[None].clone()
    v[0, 8 + 3, 0] = float("inf")
    v[0, 8 + 5, 2] = float("nan")
    v[0, 8:] += 0.25
    f = torch.cat([torch.tensor(CUBE_F), torch.tensor(CUBE_F) + 8]).to(DEV)
    v = v.to(DEV)
    o, s = torch.full((1, 3), -0.1, device=DEV), torch.full((1,), 1.5, device=DEV)
    p = ov.normalize(v, o, s)
    rows = ov.voxel_rows(p, 32, f, prune=True, split_nonfinite=False)
    out = trianglemeshes_to_voxelgrids(v, f, 32, o, s, return_sparse=True)
    assert torch.equal(out._indices(), rows.T)
    assert torch.equal(rows_of(trianglemeshes_to_voxelgrids(v, f, 32, o, s)), rows.T)


def test_nan_points_are_dropped_as_the_reference_drops_them_on_cuda():
    """The reference's quantisation, torch.round(p * (res-1)).long(), gives INT64_MIN for NaN on a CUDA
    tensor as on the CPU, so the reference drops a NaN point on both devices, and so does this library."""
    x = torch.tensor([float("nan")], device=DEV)
    assert torch.round(x * 7).long().item() == -2 ** 63
    p = torch.tensor([[[float("nan"), 0.5, 0.5], [0.2, 0.2, 0.2]]], device=DEV)
    out = pointclouds_to_voxelgrids(p, 8, torch.zeros(1, 3, device=DEV), torch.ones(1, device=DEV), return_sparse=True)
    assert out._indices().tolist() == [[0], [1], [1], [1]]


def test_bad_face_index_raises_index_error():
    v = torch.rand(2, 5, 3, device=DEV)
    for bad in (5, -1):
        f = torch.tensor([[0, 1, 2], [1, 2, bad]], device=DEV)
        with pytest.raises(IndexError, match="face 1"):
            trianglemeshes_to_voxelgrids(v, f, 16)
        with pytest.raises(IndexError):
            trianglemeshes_to_voxelgrids(v, f, 16, return_sparse=True)


def test_too_deep_face_raises_value_error():
    v = torch.tensor([[[-1e8, 0.5, 0.5], [1e8, 0.5, 0.5], [0.5, 0.7, 0.5]]], device=DEV)
    with pytest.raises(ValueError, match="levels of subdivision"):
        trianglemeshes_to_voxelgrids(v, torch.tensor([[0, 1, 2]], device=DEV), 64, torch.zeros(1, 3, device=DEV),
                                     torch.ones(1, device=DEV))


def test_empty_batch_and_no_faces():
    f = torch.tensor(CUBE_F, device=DEV)
    for sparse in (False, True):
        out = trianglemeshes_to_voxelgrids(torch.zeros((0, 8, 3), device=DEV), f, 8, return_sparse=sparse)
        assert tuple(out.shape) == (0, 8, 8, 8) and out.dtype == torch.float32
        out = pointclouds_to_voxelgrids(torch.zeros((0, 8, 3), device=DEV, dtype=torch.float64), 8,
                                        torch.zeros((0, 3), device=DEV), torch.ones(0, device=DEV), return_sparse=sparse)
        assert tuple(out.shape) == (0, 8, 8, 8) and out.dtype == torch.float64
    v = torch.tensor(CUBE_V, device=DEV)[None]
    out = trianglemeshes_to_voxelgrids(v, torch.zeros((0, 3), dtype=torch.int64, device=DEV), 8)
    assert torch.equal(out, pointclouds_to_voxelgrids(v, 8))


def test_more_than_2_31_bits_sparse():
    """B res^3 = 2.66e9 bits: a small mesh near the far corner of the second view."""
    v0, f = synthetic.icosphere(2)
    v = np.stack([v0 * 0.01 + 0.5, v0 * 0.01 + 0.985]).astype(np.float32)
    v = torch.from_numpy(v).to(DEV)
    f = torch.from_numpy(f).to(DEV)
    o, s = torch.zeros((2, 3), device=DEV), torch.ones(2, device=DEV)
    rows = check_against_oracle(v, f, 1100, o, s, dense=False)
    assert set(rows[:, 0].tolist()) == {0, 1} and int(rows[:, 1:].max()) > 1070


def count_syncs(fn):
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return len([w for w in caught if "called a synchronizing" in str(w.message)])


def test_host_reads_per_call():
    v = torch.tensor(CUBE_V, device=DEV)[None].repeat(2, 1, 1)
    f = torch.tensor(CUBE_F, device=DEV)
    o, s = torch.zeros((2, 3), device=DEV), torch.ones(2, device=DEV)
    p = torch.rand((2, 1000, 3), device=DEV)
    trianglemeshes_to_voxelgrids(v, f, 64, o, s)
    torch.cuda.synchronize()
    assert count_syncs(lambda: trianglemeshes_to_voxelgrids(v, f, 64, o, s)) == 1
    assert count_syncs(lambda: trianglemeshes_to_voxelgrids(v, f, 64, o, s, return_sparse=True)) == 1
    assert count_syncs(lambda: pointclouds_to_voxelgrids(p, 64, o, s)) == 0
    assert count_syncs(lambda: pointclouds_to_voxelgrids(p, 64, o, s, return_sparse=True)) == 1


def test_reruns_are_byte_identical():
    v0, f = synthetic.icosphere(4)
    v = torch.from_numpy(v0[None].astype(np.float32)).to(DEV)
    f = torch.from_numpy(f).to(DEV)
    a = trianglemeshes_to_voxelgrids(v, f, 200)
    b = trianglemeshes_to_voxelgrids(v, f, 200)
    assert torch.equal(a, b)
    a = trianglemeshes_to_voxelgrids(v, f, 200, return_sparse=True)
    b = trianglemeshes_to_voxelgrids(v, f, 200, return_sparse=True)
    assert torch.equal(a._indices(), b._indices())


@pytest.mark.parametrize("offset", [1, 3, 100, 255])
def test_workspace_at_an_odd_address(offset):
    B, res = 1, 64
    v = torch.tensor(CUBE_V, device=DEV)[None]
    f = torch.tensor(CUBE_F, device=DEV)
    need = _lib.voxelize_workspace_bytes(B, 12, res, "t")
    ws = torch.empty(need + offset, dtype=torch.uint8, device=DEV)
    wp = ws.data_ptr() + offset
    info = torch.empty(4, dtype=torch.int64, device=DEV)
    out = torch.empty((B, res, res, res), device=DEV)
    _lib.call("dibr_b200_voxelize_mark", DEV, B, 8, 12, res, _lib.DTYPE_F32, v, f, 1, info, wp, need)
    _lib.call("dibr_b200_voxelize_dense", DEV, B, 12, res, _lib.DTYPE_F32, out, wp, need)
    nnz = int(info[3])
    idx = torch.empty((4, nnz), dtype=torch.int64, device=DEV)
    _lib.call("dibr_b200_voxelize_sparse", DEV, B, 12, res, nnz, idx, wp, need)
    ref = trianglemeshes_to_voxelgrids(v, f, res)
    assert torch.equal(out, ref) and torch.equal(idx, rows_of(ref))
    assert _lib.lib().dibr_b200_voxelize_dense(B, 12, res, _lib.DTYPE_F32, ctypes.c_void_p(out.data_ptr()),
                                               ctypes.c_void_p(wp), need - 1, None) == _lib.EWORKSPACE


def test_peak_memory_at_512():
    v = torch.tensor(CUBE_V, device=DEV)[None]
    f = torch.tensor(CUBE_F, device=DEV)
    trianglemeshes_to_voxelgrids(v, f, 512)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = trianglemeshes_to_voxelgrids(v, f, 512)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    bits = 512 ** 3 // 8
    assert peak <= out.numel() * 4 + bits + (2 << 20), peak
    assert rows_of(out).shape[1] == 6 * 510 * 510 + 12 * 510 + 8
