"""Voxelization checks that need no GPU: the torch oracle (oracle/voxelize.py) against the reference's
own outputs stored in tests/golden/voxelize.npz, with and without the exact range prune; the public
signatures against the reference's; the workspace size query against the layout it documents; and
the argument errors raised on the host before any launch."""
import inspect
import os

import numpy as np
import pytest
import torch

from kaolin_b200 import _lib
from kaolin_b200.ops.conversions import pointclouds_to_voxelgrids, trianglemeshes_to_voxelgrids
from oracle import voxelize as ov

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "voxelize.npz")


def load_scenes():
    z = np.load(GOLDEN)
    names = sorted({k.split("/")[0] for k in z.files})
    out = {}
    for n in names:
        get = lambda k: z[f"{n}/{k}"] if f"{n}/{k}" in z.files else None
        out[n] = dict(kind=str(get("kind")), vertices=get("vertices"), faces=get("faces"), origin=get("origin"),
                      scale=get("scale"), res=int(get("res")), rows=get("rows").astype(np.int64),
                      dtype=getattr(torch, str(get("dtype"))), shape=tuple(get("shape")),
                      coalesced=bool(get("coalesced")))
    return out


SCENES = load_scenes()


def as_torch(sc, device="cpu"):
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(device)
    return t(sc["vertices"]), t(sc["faces"]), t(sc["origin"]), t(sc["scale"])


@pytest.mark.parametrize("prune", [False, True])
@pytest.mark.parametrize("name", sorted(SCENES))
def test_oracle_equals_reference_goldens(name, prune):
    sc = SCENES[name]
    v, f, o, s = as_torch(sc)
    p = ov.normalize(v, o, s)
    assert p.dtype == sc["dtype"]
    rows = ov.voxel_rows(p, sc["res"], f, prune=prune)
    np.testing.assert_array_equal(rows.T.numpy(), sc["rows"])


def test_golden_scenes_cover_the_edge_cases():
    assert len(SCENES) >= 30
    assert {"float32", "float64"} == {str(sc["dtype"]).replace("torch.", "") for sc in SCENES.values()}
    assert any(sc["faces"] is not None and sc["faces"].dtype == np.int32 for sc in SCENES.values())
    assert any(sc["vertices"].shape[0] == 3 for sc in SCENES.values())
    assert SCENES["no_faces_8"]["faces"].shape == (0, 3)


def test_signatures_match_the_reference():
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference sources absent")
    pc = ref_import.module("kaolin.ops.conversions.pointcloud")
    tm = ref_import.module("kaolin.ops.conversions.trianglemesh")
    assert inspect.signature(pointclouds_to_voxelgrids) == inspect.signature(pc.pointclouds_to_voxelgrids)
    assert inspect.signature(trianglemeshes_to_voxelgrids) == inspect.signature(tm.trianglemeshes_to_voxelgrids)


def restated_workspace(B, F, res):
    """op_layouts.h voxelize_layout: bits, counts, scan, chunk counts, chunk scan, scan tile sums, each
    from a multiple of 256 bytes, plus 256 bytes of slack for the origin."""
    up = lambda n: -(-n // 256) * 256
    nwords = -(-(B * res ** 3) // 32)
    nchunks = -(-nwords // 32)
    bf = B * F
    sizes = [4 * nwords, 4 * bf, 4 * (bf + 1), 4 * nchunks, 4 * (nchunks + 1), 4 * (-(-max(bf, nchunks) // 4096) + 1)]
    return sum(up(n) for n in sizes[:-1]) + sizes[-1] + 256


@pytest.mark.parametrize("B,F,res", [(1, 12, 2), (1, 0, 3), (3, 1280, 128), (8, 81920, 512), (2, 12, 1100),
                                     (0, 5, 64), (5, 7, 1), (1, 1, 1 << 20)])
def test_workspace_size_query_matches_the_layout(B, F, res):
    if B * res ** 3 // 1024 >= 2 ** 31 - 1:
        with pytest.raises(RuntimeError):
            _lib.voxelize_workspace_bytes(B, F, res, "q")
        return
    assert _lib.voxelize_workspace_bytes(B, F, res, "q") == restated_workspace(B, F, res)


def test_size_limits_and_bad_arguments_on_the_host():
    lib = _lib.lib()
    import ctypes
    n = ctypes.c_size_t(0)
    assert lib.dibr_b200_voxelize_workspace_bytes(-1, 1, 8, ctypes.byref(n)) == _lib.EINVAL
    assert lib.dibr_b200_voxelize_workspace_bytes(1, 1, 0, ctypes.byref(n)) == _lib.EINVAL
    assert lib.dibr_b200_voxelize_workspace_bytes(1, 2 ** 31, 8, ctypes.byref(n)) == _lib.ESIZE
    assert lib.dibr_b200_voxelize_workspace_bytes(1, 1, (1 << 20) + 1, ctypes.byref(n)) == _lib.ESIZE
    # NULL info, bad dtype and a short workspace are refused before any launch
    assert lib.dibr_b200_voxelize_mark(1, 3, 0, 8, 0, 4096, None, 0, None, 4096, 1 << 20, None) == _lib.EINVAL
    assert lib.dibr_b200_voxelize_mark(1, 3, 0, 8, 5, 4096, None, 0, 4096, 4096, 1 << 20, None) == _lib.EINVAL
    assert lib.dibr_b200_voxelize_mark(1, 3, 1, 8, 0, 4096, None, 0, 4096, 4096, 1 << 20, None) == _lib.EINVAL
    need = _lib.voxelize_workspace_bytes(1, 0, 8, "q")
    assert lib.dibr_b200_voxelize_mark(1, 3, 0, 8, 0, 4096, None, 0, 4096, 4097, need - 1, None) == _lib.EWORKSPACE
    assert lib.dibr_b200_voxelize_dense(1, 0, 8, 0, 4104, 4096, need, None) == _lib.EINVAL     # misaligned output
    assert lib.dibr_b200_voxelize_sparse(1, 0, 8, 2 ** 31, 4096, 4096, need, None) == _lib.ESIZE


def test_python_errors_are_raised_before_any_launch():
    v = torch.rand(1, 4, 3)
    f = torch.tensor([[0, 1, 2]])
    with pytest.raises(TypeError):
        trianglemeshes_to_voxelgrids(v, f, 8.0)
    with pytest.raises(TypeError):
        pointclouds_to_voxelgrids(v, 8.0)
    with pytest.raises(NotImplementedError):
        trianglemeshes_to_voxelgrids(v, f, 8)
    with pytest.raises(NotImplementedError):
        pointclouds_to_voxelgrids(v, 8)
    for res in (1, 0, -3):
        with pytest.raises(ValueError):
            trianglemeshes_to_voxelgrids(v, f, res)
    with pytest.raises(ValueError):
        pointclouds_to_voxelgrids(v, 0)
