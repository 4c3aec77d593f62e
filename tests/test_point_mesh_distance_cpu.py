"""point_to_mesh_distance without a GPU: the float64 oracle (oracle/point_mesh_distance.py) against the
reference operator's stored outputs, the workspace layout of the new op_layouts.h family, and the
argument checks of the public function, of ``_C.metrics`` and of the C ABI."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import point_mesh_distance as oracle
from oracle import ref_golden_point_mesh as golden
from kaolin_b200 import _C, _lib
from kaolin_b200.metrics import point_to_mesh_distance

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host_math", "point_mesh_layout.cpp")
HDR = os.path.join(ROOT, "kaolin_b200", "csrc", "op_layouts.h")
LIB = os.path.join(ROOT, "tests", "host_math", "_build", "point_mesh_layout.so")
ALIGN = 256
INT32_MAX = 2 ** 31 - 1
SCENES = golden.scenes()
STORED = golden.load()


def test_every_scene_has_stored_reference_outputs():
    assert set(STORED) == {(n, dt) for n in SCENES for dt in golden.DTYPES}
    for key, out in STORED.items():
        assert set(out) == set(golden.OUTPUTS), key


# Rows where the oracle's nearest face or type may legitimately differ from the reference's: the
# reference's result is within the float32 bound of another face's (or region's) distance.
TIE_SCENES = {"docstring", "exact", "duplicates", "fan", "tiles_511", "tiles_512", "tiles_513", "tiles_1025"}


@pytest.mark.parametrize("scene", sorted(SCENES))
def test_oracle_agrees_with_stored_reference(scene):
    points, faces, _ = SCENES[scene]
    ref = STORED[(scene, "f64")]
    for b in range(points.shape[0]):
        p, fv = points[b], faces[b]
        finite = np.isfinite(p).all(1) & (np.abs(p) < 1e30).all(1)
        if not (np.isfinite(fv).all() and (np.abs(fv) < 1e30).all()) or scene.startswith("degenerate"):
            continue   # the oracle has no answer for NaN, inf or degenerate faces
        d, f, t = oracle.numpy_distance(p[finite], fv)
        rd = ref["dist"][b][finite]
        # float32 bound: the reference rounds dist to float; the pair arithmetic adds a few ulps of |p|^2
        scale = 1.0 + (p[finite] ** 2).sum(1) + (fv ** 2).sum((1, 2)).max()
        assert np.all(np.abs(rd - d) <= 1e-5 * scale), scene
        same = (f == ref["face_idx"][b][finite]) & (t == ref["dist_type"][b][finite])
        if scene not in TIE_SCENES:
            assert same.mean() >= 0.99, (scene, same.mean())


def test_docstring_example_is_stored():
    ref = STORED[("docstring", "f32")]
    np.testing.assert_array_equal(ref["dist"], np.array([[0.25, 41.0]], np.float32))
    np.testing.assert_array_equal(ref["face_idx"], [[0, 0]])
    np.testing.assert_array_equal(ref["dist_type"], [[5, 5]])


def test_types_scene_reaches_every_type():
    for dt in golden.DTYPES:
        np.testing.assert_array_equal(STORED[("types", dt)]["dist_type"][0], np.arange(7))


@pytest.fixture(scope="module")
def pm():
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(SRC), os.path.getmtime(HDR)):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", LIB, SRC])
    lib = ctypes.CDLL(LIB)
    lib.pm_layout.argtypes = [ctypes.c_int] * 4 + [ctypes.c_int64, ctypes.POINTER(ctypes.c_int64)]
    lib.pm_carve.argtypes = [ctypes.c_uint64] * 3
    lib.pm_carve.restype = ctypes.c_int64
    return lib


FWD = ("records", "keys")
BWD = ("terms", "count", "off", "sums", "ids", "long_rows", "long_count")
SHAPES = [(1, 0, 0), (1, 1, 1), (0, 5, 5), (2, 2048, 1280), (3, 100000, 81920), (1, 4097, 4097),
          (1, INT32_MAX - 1, 1), (1, 1, INT32_MAX - 1), (8, 250000, 20480)]


def needs(backward, B, N, F, ts):
    """Bytes each piece's kernels index."""
    np_, nf = B * N, B * F
    if not backward:
        return {"records": nf * 33 * ts, "keys": np_ * 8}
    return {"terms": np_ * 9 * ts, "count": nf * 4, "off": (nf + 1) * 4, "sums": 4 * ((nf + 4095) // 4096 + 1),
            "ids": np_ * 4, "long_rows": nf * 4, "long_count": 4}


@pytest.mark.parametrize("backward", [0, 1])
def test_layout_pieces_are_aligned_apart_and_inside(pm, backward):
    names = BWD if backward else FWD
    for B, N, F in SHAPES:
        for ts in (4, 8):
            out = (ctypes.c_int64 * 32)()
            assert pm.pm_layout(backward, B, N, F, ts, out) == 1 + 2 * len(names)
            total = out[0]
            pieces = {n: (out[1 + 2 * i], out[2 + 2 * i]) for i, n in enumerate(names)}
            for name, need in needs(backward, B, N, F, ts).items():
                assert pieces[name][1] >= need, (B, N, F, ts, name)
            spans = sorted((at, at + n) for at, n in pieces.values() if n > 0)
            for (_, e0), (s1, _) in zip(spans, spans[1:]):
                assert e0 <= s1
            for offset in (0, 1, 3, 8, 255):
                ws = 0x10000 + offset
                origin = pm.pm_carve(ws, total, total)
                assert 0 <= origin < ALIGN and (ws + origin) % ALIGN == 0
                for at, n in pieces.values():
                    assert (ws + origin + at) % ALIGN == 0 and origin + at + n <= total
                assert pm.pm_carve(ws, total - 1, total) == -1


def test_size_query_returns_the_header_totals(pm):
    for B, N, F in [(1, 1, 1), (2, 2048, 1280), (3, 1000, 0), (1, 0, 7)]:
        for dtype, ts in ((_lib.DTYPE_F32, 4), (_lib.DTYPE_F64, 8)):
            fwd, bwd = _lib.point_mesh_distance_workspace_bytes(B, N, F, dtype, "q")
            for backward, got in ((0, fwd), (1, bwd)):
                out = (ctypes.c_int64 * 32)()
                pm.pm_layout(backward, B, N, F, ts, out)
                assert got == out[0]


def test_c_abi_size_limits_and_arguments():
    lib = _lib.lib()
    f, b = ctypes.c_size_t(0), ctypes.c_size_t(0)
    q = lib.dibr_b200_point_mesh_distance_workspace_bytes
    assert q(1, INT32_MAX, 1, _lib.DTYPE_F32, ctypes.byref(f), ctypes.byref(b)) == _lib.ESIZE
    assert q(2, 2 ** 30, 1, _lib.DTYPE_F32, ctypes.byref(f), ctypes.byref(b)) == _lib.ESIZE
    assert q(1, 1, INT32_MAX, _lib.DTYPE_F64, ctypes.byref(f), ctypes.byref(b)) == _lib.ESIZE
    assert q(1, INT32_MAX - 1, 1, _lib.DTYPE_F32, ctypes.byref(f), ctypes.byref(b)) == 0
    assert q(1, 1, 1, 7, ctypes.byref(f), ctypes.byref(b)) == _lib.EINVAL
    assert q(-1, 1, 1, _lib.DTYPE_F32, ctypes.byref(f), ctypes.byref(b)) == _lib.EINVAL
    assert lib.dibr_b200_point_mesh_distance_forward(1, 1, 1, _lib.DTYPE_F32, 1, 1, 1, 1, 1, None, 1 << 20,
                                                     None) == _lib.EINVAL
    q(1, 16, 16, _lib.DTYPE_F32, ctypes.byref(f), ctypes.byref(b))
    buf = ctypes.create_string_buffer(f.value + 300)
    for off in (0, 1, 7):
        ws = ctypes.addressof(buf) + off
        assert lib.dibr_b200_point_mesh_distance_forward(1, 16, 16, _lib.DTYPE_F32, 1, 1, 1, 1, 1, ws, f.value - 1,
                                                         None) == _lib.EWORKSPACE
        assert lib.dibr_b200_point_mesh_distance_backward(1, 16, 16, _lib.DTYPE_F32, 1, 1, 1, 1, 1, 1, 1, ws,
                                                          b.value - 1, None) == _lib.EWORKSPACE


def test_public_function_argument_checks():
    p, fv = torch.zeros(1, 4, 3), torch.zeros(1, 2, 3, 3)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        point_to_mesh_distance(p, fv)
    with pytest.raises(TypeError):
        point_to_mesh_distance(p.numpy(), fv)


def test_c_metrics_namespace_and_checks():
    fwd = _C.metrics.unbatched_triangle_distance_forward_cuda
    bwd = _C.metrics.unbatched_triangle_distance_backward_cuda
    assert fwd.__code__.co_argcount == 5 and bwd.__code__.co_argcount == 7
    p, fv = torch.zeros(4, 3), torch.zeros(2, 3, 3)
    d, i, t = torch.zeros(4), torch.zeros(4, dtype=torch.long), torch.zeros(4, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="points must be a CUDA tensor"):
        fwd(p, fv, d, i, t)
    with pytest.raises(RuntimeError, match="grad_dist must be a CUDA tensor"):
        bwd(d, p, fv, i, t, torch.zeros_like(p), torch.zeros_like(fv))
