"""voxelgrids_to_cubic_meshes without a GPU: the numpy oracle (oracle/cubic_meshes.py) against every
output of the reference stored in tests/golden/cubic_meshes.npz, the workspace layout, and the C ABI's
host-side argument and size errors."""
import ctypes
import inspect
import os
import subprocess

import numpy as np
import pytest
import torch

from kaolin_b200 import _lib
from kaolin_b200.ops import conversions
from oracle import cubic_meshes as O

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "cubic_meshes.npz")
SRC = os.path.join(ROOT, "tests", "host_math", "cubic_meshes_layout.cpp")
HDR = os.path.join(ROOT, "kaolin_b200", "csrc", "op_layouts.h")
LIB = os.path.join(ROOT, "tests", "host_math", "_build", "cubic_meshes_layout.so")
ALIGN = 256
INT32_MAX = 2 ** 31 - 1

_G = np.load(GOLDEN)
SCENES = sorted({k.split("__")[0] for k in _G.files})
MODES = {"tri": True, "quad": False}


def golden(name, mode):
    """(grid, [vertices], [faces int64]) of one scene in one mode."""
    grid = _G[f"{name}__grid"]
    return (grid, [_G[f"{name}__{mode}__v{b}"] for b in range(grid.shape[0])],
            [_G[f"{name}__{mode}__f{b}"].astype(np.int64) for b in range(grid.shape[0])])


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", SCENES)
def test_oracle_equals_reference(name, mode):
    grid, rv, rf = golden(name, mode)
    ov, of = O.cubic_meshes(grid, MODES[mode])
    for b in range(grid.shape[0]):
        assert ov[b].dtype == np.float32 and of[b].dtype == np.int64
        assert ov[b].shape == rv[b].shape and np.array_equal(ov[b], rv[b]), (name, mode, b)
        assert of[b].shape == rf[b].shape and np.array_equal(of[b], rf[b]), (name, mode, b)


def test_goldens_cover_the_scenes_that_matter():
    _, v, f = golden("single_voxel", "tri")
    assert v[0].shape == (8, 3) and f[0].shape == (12, 3)
    _, v, f = golden("box_3x4x5", "quad")
    assert f[0].shape == (2 * (12 + 20 + 15), 4) and v[0].shape == (4 * 5 * 6 - 2 * 3 * 4, 3)
    _, v, f = golden("fixture", "quad")
    assert v[0].shape == (0, 3) and f[0].shape == (0, 4) and all(len(x) for x in f[1:])
    _, v, f = golden("batch4_empty_view1", "tri")
    assert f[1].shape == (0, 3) and all(len(x) for x in f[::2])
    # differences of 1/2 round to no face: the quarter grid has fewer faces than its occupancy
    grid, _, f = golden("quarters_f32", "quad")
    occupied = O.cubic_meshes(grid != 0, False)[1]
    assert sum(len(x) for x in f) < sum(len(x) for x in occupied)
    for dt in ("bool", "u8", "f32"):
        assert _G[f"binary_{dt}__grid"].dtype == {"bool": np.bool_, "u8": np.uint8, "f32": np.float32}[dt]


def test_oracle_winds_by_the_sign_of_the_difference():
    """0/255 gives the 0/1 result; the reference would reverse only where d == -1."""
    rng = np.random.default_rng(5)
    g = rng.random((6, 7, 5)) < 0.5
    for tri in (True, False):
        v1, f1 = O.extract(g.astype(np.uint8), tri)
        v2, f2 = O.extract(g.astype(np.uint8) * 255, tri)
        assert np.array_equal(v1, v2) and np.array_equal(f1, f2)
    v, f = O.extract(np.array([[[1.0, np.nan, 0.0, 0.4, 2.5]]], np.float32), False)
    # x and y: two faces each for the voxels 1, NaN and 2.5 (0.4 rounds to 0); z: at z = 0, 1, 2, 4, 5
    assert len(f) == 6 + 6 + 5 and len(v) == 4 * 5            # no corner at z = 3


def test_signature_and_cpu_input():
    assert str(inspect.signature(conversions.voxelgrids_to_cubic_meshes)) == "(voxelgrids, is_trimesh=True)"
    with pytest.raises(NotImplementedError, match="does not support CPU"):
        conversions.voxelgrids_to_cubic_meshes(torch.ones(1, 2, 2, 2))


# ---------------------------------------------------------------------------------------------
# Workspace layout and the C ABI's host-side checks.

@pytest.fixture(scope="module")
def lay():
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(SRC), os.path.getmtime(HDR)):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", LIB, SRC])
    lib = ctypes.CDLL(LIB)
    lib.cm_layout.argtypes = [ctypes.c_int64, ctypes.c_int64, ctypes.POINTER(ctypes.c_int64)]
    lib.cm_carve.argtypes = [ctypes.c_uint64] * 3
    lib.cm_carve.restype = ctypes.c_int64
    return lib


SHAPES = [(1, 1, 1, 1), (2, 3, 4, 5), (5, 31, 1, 1), (3, 30, 1, 1), (8, 256, 256, 256), (2, 128, 64, 32),
          (1000, 2, 2, 2), (1, 811, 811, 811)]


@pytest.mark.parametrize("shape", SHAPES)
def test_layout_pieces_alignment_and_carve(lay, shape):
    B, X, Y, Z = shape
    L = (X + 1) * (Y + 1) * (Z + 1)
    out = (ctypes.c_int64 * 10)()
    lay.cm_layout(B, L, out)
    total, W = out[0], out[1]
    pieces = [(out[2 + 2 * i], out[3 + 2 * i]) for i in range(4)]
    assert W == -(-L // 32)
    n = 4 * B * W
    assert [p[1] for p in pieces] == [4 * 7 * B * W, 4 * n, 4 * (n + 1), 4 * (-(-n // 4096) + 1)]
    assert pieces[0][0] == 0
    for (a, na), (b, _) in zip(pieces, pieces[1:]):
        assert b == -(-(a + na) // ALIGN) * ALIGN          # back to back, each from a multiple of 256
    assert total == pieces[-1][0] + pieces[-1][1] + ALIGN
    for offset in (0, 1, 3, 8, 255):
        ws = 0x10000 + offset
        origin = lay.cm_carve(ws, total, total)
        assert 0 <= origin < ALIGN and (ws + origin) % ALIGN == 0
        assert all((ws + origin + at) % ALIGN == 0 and origin + at + nb <= total for at, nb in pieces)
        assert lay.cm_carve(ws, total - 1, total) == -1
    assert lay.cm_carve(0, total, total) == -1
    assert _lib.cubic_meshes_workspace_bytes(B, X, Y, Z, "q") == total


def _ws(B, X, Y, Z):
    n = ctypes.c_size_t(0)
    return _lib.lib().dibr_b200_cubic_meshes_workspace_bytes(B, X, Y, Z, ctypes.byref(n))


def test_c_abi_size_limits():
    # 4 B (X+1)(Y+1)(Z+1) must stay below 2^31 - 1: B L < 2^29 = 536 870 912
    assert _ws(1, 811, 811, 811) == 0                       # 812^3 = 535 387 328
    assert _ws(1, 812, 812, 812) == _lib.ESIZE              # 813^3 = 537 367 797
    assert _ws(2 ** 26, 1, 1, 1) == _lib.ESIZE              # 8 B = 2^29
    assert _ws(2 ** 26 - 1, 1, 1, 1) == 0
    assert _ws(8, 255, 255, 255) == 0 and _ws(32, 255, 255, 255) == _lib.ESIZE
    assert _ws(0, 2 ** 16, 2 ** 15, 1) == _lib.ESIZE        # one view's lattice above 2^31 - 1
    assert _ws(0, INT32_MAX, 1, 1) == _lib.ESIZE
    assert _ws(0, 2 ** 40, 2 ** 40, 2 ** 40) == _lib.ESIZE   # no wrap in the lattice product
    assert _ws(2 ** 40, 2, 2, 2) == _lib.ESIZE
    assert _ws(0, 5, 5, 5) == 0
    with pytest.raises(RuntimeError, match="index overflow"):
        _lib.cubic_meshes_workspace_bytes(1, 812, 812, 812, "voxelgrids_to_cubic_meshes")


def test_c_abi_rejects_bad_arguments_before_any_launch():
    lib = _lib.lib()
    n = ctypes.c_size_t(0)
    assert lib.dibr_b200_cubic_meshes_workspace_bytes(1, 2, 2, 2, None) == _lib.EINVAL
    for args in ((-1, 2, 2, 2), (1, 0, 2, 2), (1, 2, -3, 2), (1, 2, 2, 0)):
        assert lib.dibr_b200_cubic_meshes_workspace_bytes(*args, ctypes.byref(n)) == _lib.EINVAL, args
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.cast(buf, ctypes.c_void_p).value
    strides = (8, 4, 2, 1)

    def count(B=1, dtype=_lib.DTYPE_F32, grid=p, totals=p, ws=p, nbytes=1 << 16, size=2):
        return lib.dibr_b200_cubic_meshes_count(B, size, size, size, dtype, grid, *strides, totals, ws, nbytes, None)

    assert count(dtype=_lib.DTYPE_F64) == _lib.EINVAL
    assert count(dtype=_lib.DTYPE_BOOL) == _lib.EINVAL
    for kw in ("grid", "totals", "ws"):
        assert count(**{kw: None}) == _lib.EINVAL, kw
    assert count(nbytes=16) == _lib.EWORKSPACE
    assert count(B=1 << 30) == _lib.ESIZE
    assert count(size=812) == _lib.ESIZE
    assert count(B=-1) == _lib.EINVAL

    def emit(B=1, verts=p, faces=p, ws=p, nbytes=1 << 16):
        return lib.dibr_b200_cubic_meshes_emit(B, 2, 2, 2, 1, verts, faces, ws, nbytes, None)

    for kw in ("verts", "faces", "ws"):
        assert emit(**{kw: None}) == _lib.EINVAL, kw
    assert emit(nbytes=16) == _lib.EWORKSPACE
    assert emit(B=1 << 30) == _lib.ESIZE
