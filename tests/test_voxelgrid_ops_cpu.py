"""kaolin.ops.voxelgrid without a GPU: the numpy oracle (oracle/voxelgrid.py) against every output of the
reference stored in tests/golden/voxelgrid.npz, the fill workspace layout, and the C ABI's host-side
argument and size errors."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from kaolin_b200 import _lib
from kaolin_b200.ops import voxelgrid as vg
from oracle import voxelgrid as ov

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "voxelgrid.npz")
SRC = os.path.join(ROOT, "tests", "host_math", "voxelgrid_layout.cpp")
HDR = os.path.join(ROOT, "kaolin_b200", "csrc", "op_layouts.h")
LIB = os.path.join(ROOT, "tests", "host_math", "_build", "voxelgrid_layout.so")
ALIGN = 256
INT32_MAX = 2 ** 31 - 1

_G = np.load(GOLDEN)


def scenes(func):
    """{scene: {item: array}} of one function's goldens."""
    out = {}
    for k in _G.files:
        f, name, item = k.split("__")
        if f == func:
            out.setdefault(name, {})[item] = _G[k]
    return out


FILL, SURFACE, ODMS, PROJECT = scenes("fill"), scenes("surface"), scenes("odms"), scenes("project")


def project_args(sc):
    return sc["odms"], sc.get("grid"), int(sc["votes"])


@pytest.mark.parametrize("name", sorted(FILL))
def test_oracle_fill_equals_reference(name):
    np.testing.assert_array_equal(ov.fill(FILL[name]["grid"]), FILL[name]["out"])


@pytest.mark.parametrize("mode", ["wide", "thin"])
@pytest.mark.parametrize("name", sorted(SURFACE))
def test_oracle_surface_equals_reference(name, mode):
    np.testing.assert_array_equal(ov.extract_surface(SURFACE[name]["grid"], mode), SURFACE[name][mode])


@pytest.mark.parametrize("name", sorted(ODMS))
def test_oracle_odms_equals_reference(name):
    np.testing.assert_array_equal(ov.extract_odms(ODMS[name]["grid"]), ODMS[name]["out"])


@pytest.mark.parametrize("name", sorted(PROJECT))
def test_oracle_project_equals_reference(name):
    np.testing.assert_array_equal(ov.project_odms(*project_args(PROJECT[name])), PROJECT[name]["out"])


def test_goldens_cover_the_scenes_that_matter():
    """The fill goldens include cavities that are and are not filled, and the uint8 wrap is stored."""
    filled = {n: int((s["out"] & ~(s["grid"] != 0)).sum()) for n, s in FILL.items()}
    assert filled["cavity"] > 0 and filled["leak_edge"] > 0 and filled["leak_corner"] > 0
    assert filled["hole_to_border"] == 0 and filled["serpentine"] == 0 and filled["spiral"] == 0
    assert (~FILL["serpentine"]["out"]).sum() > 100 and (~FILL["spiral"]["out"]).sum() > 100
    u8 = PROJECT["u8_wrap_i32_v1"]
    as_bool = ov.project_odms(u8["odms"], u8["grid"].astype(bool), 1)
    assert (u8["out"] & ~as_bool).any()     # v = 1, votes = 1 and a count of 2 or more wrap to true


def test_every_function_refuses_cpu_tensors():
    g = torch.ones((1, 3, 3, 3))
    for f in (vg.fill, vg.extract_surface, vg.extract_odms, vg.project_odms, lambda t: vg.downsample(t, 2)):
        with pytest.raises(NotImplementedError):
            f(g if f is not vg.project_odms else torch.zeros((1, 6, 3, 3)))


# ---------------------------------------------------------------------------------------------
# Workspace layout and the C ABI's host-side checks.

@pytest.fixture(scope="module")
def lay():
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(SRC), os.path.getmtime(HDR)):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", LIB, SRC])
    lib = ctypes.CDLL(LIB)
    lib.vg_layout.argtypes = [ctypes.c_int64, ctypes.c_int64, ctypes.POINTER(ctypes.c_int64)]
    lib.vg_carve.argtypes = [ctypes.c_uint64] * 3
    lib.vg_carve.restype = ctypes.c_int64
    return lib


SHAPES = [(1, 1, 1, 1), (2, 5, 7, 9), (8, 256, 256, 256), (1, 1024, 1024, 1024), (1000, 3, 3, 3),
          (3, 1290, 1290, 1290)]


def test_fill_layout_is_four_bytes_per_voxel_and_aligned(lay):
    for B, X, Y, Z in SHAPES:
        out = (ctypes.c_int64 * 3)()
        lay.vg_layout(B, X * Y * Z, out)
        total, at, n = out
        assert n == 4 * B * X * Y * Z and total <= n + ALIGN
        for offset in (0, 1, 3, 8, 255):
            ws = 0x10000 + offset
            origin = lay.vg_carve(ws, total, total)
            assert 0 <= origin < ALIGN and (ws + origin + at) % ALIGN == 0 and origin + at + n <= total
            assert lay.vg_carve(ws, total - 1, total) == -1
        assert _lib.voxelgrid_fill_workspace_bytes(B, X, Y, Z, "q") == total


def test_c_abi_size_limits_and_arguments():
    lib = _lib.lib()
    n = ctypes.c_size_t(0)
    q = lib.dibr_b200_voxelgrid_fill_workspace_bytes
    assert q(1, 1290, 1290, 1290, ctypes.byref(n)) == 0                  # 2 146 689 000 voxels
    assert q(1, 1291, 1291, 1291, ctypes.byref(n)) == _lib.ESIZE
    assert q(1, 2 ** 16, 2 ** 15, 1, ctypes.byref(n)) == _lib.ESIZE      # exactly 2^31
    assert q(1, INT32_MAX - 1, 1, 1, ctypes.byref(n)) == 0
    assert q(10 ** 9, 1290, 1290, 1290, ctypes.byref(n)) == _lib.ESIZE   # the labels overflow
    assert q(-1, 2, 2, 2, ctypes.byref(n)) == _lib.EINVAL
    assert q(1, 2, -2, 2, ctypes.byref(n)) == _lib.EINVAL
    assert q(0, 2, 2, 2, ctypes.byref(n)) == 0
    assert q(1, 2, 2, 2, None) == _lib.EINVAL
    with pytest.raises(RuntimeError):
        _lib.voxelgrid_fill_workspace_bytes(1, 1291, 1291, 1291, "fill")
    # NULL buffers, bad dtypes and a misaligned output are rejected on the host, before any launch
    F32, U8 = _lib.DTYPE_F32, _lib.DTYPE_U8
    fill = lib.dibr_b200_voxelgrid_fill
    assert fill(1, 4, 4, 4, F32, None, 64, 16, 4, 1, None, None, 0, None) == _lib.EINVAL
    assert fill(1, 4, 4, 4, _lib.DTYPE_F64, 4096, 64, 16, 4, 1, 4096, 4096, 1 << 20, None) == _lib.EINVAL
    assert fill(1, 4, 4, 4, U8, 4096, 64, 16, 4, 1, 4097, 4096, 1 << 20, None) == _lib.EINVAL
    assert fill(1, 4, 4, 4, U8, 4096, 64, 16, 4, 1, 4096, 4096, 16, None) == _lib.EWORKSPACE
    assert fill(1, 1291, 1291, 1291, U8, 4096, 0, 0, 0, 0, 4096, 4096, 16, None) == _lib.ESIZE
    assert fill(0, 4, 4, 4, U8, None, 64, 16, 4, 1, None, None, 0, None) == 0          # nothing to do
    surf = lib.dibr_b200_voxelgrid_extract_surface
    assert surf(1, 4, 4, 4, F32, 0, None, 64, 16, 4, 1, None, None) == _lib.EINVAL
    assert surf(1, 4, 4, 4, _lib.DTYPE_I32, 0, 4096, 64, 16, 4, 1, 4096, None) == _lib.EINVAL
    assert surf(1, 1291, 1291, 1291, F32, 0, 4096, 0, 0, 0, 0, 4096, None) == _lib.ESIZE
    odms = lib.dibr_b200_voxelgrid_extract_odms
    assert odms(1, 4, F32, None, 64, 16, 4, 1, None, None) == _lib.EINVAL
    assert odms(1, 4, _lib.DTYPE_F64, 4096, 64, 16, 4, 1, 4096, None) == _lib.EINVAL
    proj = lib.dibr_b200_voxelgrid_project_odms
    ones = _lib.VOXELGRID_ALL_ONES
    assert proj(1, 4, _lib.DTYPE_I64, None, ones, None, 0, 0, 0, 0, 1, 4096, None) == _lib.EINVAL
    assert proj(1, 4, _lib.DTYPE_U8, 4096, ones, None, 0, 0, 0, 0, 1, 4096, None) == _lib.EINVAL
    assert proj(1, 4, _lib.DTYPE_I64, 4096, _lib.DTYPE_BOOL, None, 0, 0, 0, 0, 1, 4096, None) == _lib.EINVAL
    assert proj(1, 4, _lib.DTYPE_I64, 4096, 9, 4096, 0, 0, 0, 0, 1, 4096, None) == _lib.EINVAL
    assert proj(1, 1291, _lib.DTYPE_I64, 4096, ones, None, 0, 0, 0, 0, 1, 4096, None) == _lib.ESIZE
