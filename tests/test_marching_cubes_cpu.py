"""Marching cubes without a GPU: the numpy restatement (oracle/marching_cubes.py), corrected and
faithful, against the reference's own outputs (tests/golden/ref_cuda_mcube.npz); the library's case table against the one
read off the reference's outputs; the public signatures; argument errors; and the C entry points' EINVAL / ESIZE returns."""
import ctypes
import functools
import inspect

import numpy as np
import pytest
import torch

from kaolin_b200 import _C, _lib
from kaolin_b200.ops import conversions
from oracle import marching_cubes as O
from oracle import ref_golden_mcube


def reference(name, scenes=O.SCENES):
    grid, iso = scenes[name][0](), scenes[name][1]
    return grid, iso, ref_golden_mcube.reference(name, None, [])


@functools.lru_cache(None)
def tables():
    """The oracle's case tables, read off the reference's outputs for the 256 corner configurations."""
    _, _, ref = reference("cases")
    return O.Tables(O.case_table_from_golden(
        [(ref_golden_mcube.rows(ref, f"v{k}")[1], ref_golden_mcube.rows(ref, f"f{k}")[1]) for k in range(256)]))


@pytest.mark.parametrize("name", list(O.SCENES))
def test_oracle_reproduces_reference(name):
    grid, iso, ref = reference(name)
    for b in range(grid.shape[0]):
        v, f, _ = O.extract(grid[b], iso, tables())
        for key, ours in ((f"v{b}", v), (f"f{b}", f)):
            rows, values = ref_golden_mcube.rows(ref, key)
            assert tuple(ours.shape) == tuple(ref._entry(key)["shape"]), (name, key)
            assert O.same_bits(ours[rows], values), (name, key)
            if not np.isnan(ours).any():
                assert ref.equal(key, ours), (name, key)


@pytest.mark.parametrize("name", list(O.QUIRKS))
def test_faithful_oracle_reproduces_reference_quirks(name):
    """The faithful restatement reproduces the reference's wrong outputs (dropped voxels, scrambled
    strides, vertex cap), except at face corners where the reference reads an uninitialised offset;
    the corrected one differs from them."""
    grid, iso, ref = reference(name, O.QUIRKS)
    v, f, _ = O.extract(grid[0], iso, tables(), faithful=True)
    assert (f != -3).all()
    rows, values = ref_golden_mcube.rows(ref, "v0")
    assert tuple(v.shape) == tuple(ref._entry("v0")["shape"]) and O.same_bits(v[rows], values)
    rows, values = ref_golden_mcube.rows(ref, "f0")
    assert tuple(f.shape) == tuple(ref._entry("f0")["shape"])
    defined = f[rows] != -2
    assert defined.mean() > 0.9 and np.array_equal(f[rows][defined], values[defined])
    if (f != -2).all():
        assert ref.equal("f0", f)
    cv, cf, _ = O.extract(grid[0], iso, tables())
    assert not (ref.equal("v0", cv) and ref.equal("f0", cf))


def test_library_case_table_equals_reference():
    ours = conversions.voxelgrid.case_table().numpy()
    for cs in range(256):
        pairs = [tuple(p) for p in ours[cs].reshape(-1, 2) if p[0] >= 0]
        assert all(p[1] >= 0 for p in pairs)
        assert [O.EDGES.index(p) for p in pairs] == tables().table[cs], cs
        inside = [(cs >> k) & 1 for k in range(8)]
        # every triangle vertex lies on a sign-change edge, and every sign-change edge is used
        assert all(inside[i] != inside[j] for i, j in pairs), cs
        assert set(pairs) == {e for e in O.EDGES if inside[e[0]] != inside[e[1]]}, cs
        assert len(pairs) % 3 == 0 and (ours[cs].reshape(-1, 2)[len(pairs):] == -1).all()


def test_signatures_match_reference():
    assert str(inspect.signature(conversions.voxelgrids_to_trianglemeshes)) == "(voxelgrids, iso_value=0.5)"
    assert str(inspect.signature(_C.ops.conversions.unbatched_mcube_forward_cuda)) == "(voxelgrid, iso_value)"


def test_argument_errors():
    with pytest.raises(NotImplementedError, match="does not support CPU"):
        conversions.voxelgrids_to_trianglemeshes(torch.ones(1, 2, 2, 2))
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.ops.conversions.unbatched_mcube_forward_cuda(torch.ones(2, 2, 2), 0.5)


def _ws(B, X, Y, Z, pad):
    out = ctypes.c_size_t(0)
    return _lib.lib().dibr_b200_marching_cubes_workspace_bytes(B, X, Y, Z, pad, ctypes.byref(out)), out.value


def test_aligned_workspace_bytes_and_size_limits():
    status, nbytes = _ws(2, 256, 256, 256, 1)
    cubes = 2 * 258 ** 3
    align = lambda v: (v + 255) // 256 * 256
    # the counts, the scan's tile sums from the next 256-byte boundary, and 256 bytes to align the pointer
    assert status == 0 and nbytes == align(8 * cubes) + 4 * (-(-cubes // 4096) + 1) + 256
    assert _ws(0, 3, 3, 3, 1) == (0, 4 + 256)
    for args in ((-1, 2, 2, 2, 1), (1, 0, 2, 2, 1), (1, 2, -3, 2, 0), (1, 2, 2, 2, 2)):
        assert _ws(*args)[0] == _lib.EINVAL, args
    # B * (X + 2)^3 must not exceed (2^31 - 1) // 5 = 429 496 729: 754^3 fits, 755^3 does not
    assert _ws(1, 752, 752, 752, 1)[0] == 0
    assert _ws(1, 753, 753, 753, 1)[0] == _lib.ESIZE
    assert _ws(1, 754, 754, 754, 0)[0] == 0
    assert _ws(26, 256, 256, 256, 1)[0] == _lib.ESIZE
    assert _ws(25, 256, 256, 256, 1)[0] == 0
    assert _lib.lib().dibr_b200_marching_cubes_workspace_bytes(1, 2, 2, 2, 1, None) == _lib.EINVAL


def test_entry_points_reject_bad_arguments_before_any_launch():
    lib = _lib.lib()
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.cast(buf, ctypes.c_void_p).value
    strides = (8, 4, 2, 1)
    count = lambda B=1, pad=1, dtype=_lib.DTYPE_F32, grid=p, cases=p, scan=p, totals=p, ws=p, nbytes=1 << 16: (
        lib.dibr_b200_marching_cubes_count(B, 2, 2, 2, pad, dtype, grid, *strides, 0.5, cases, scan, totals, ws, nbytes,
                                           None))
    assert count(dtype=_lib.DTYPE_F64) == _lib.EINVAL
    assert count(pad=3) == _lib.EINVAL
    for kw in ("grid", "cases", "scan", "totals", "ws"):
        assert count(**{kw: None}) == _lib.EINVAL, kw
    assert count(nbytes=16) == _lib.EWORKSPACE
    assert count(B=1 << 30) == _lib.ESIZE
    emit = lambda **kw: lib.dibr_b200_marching_cubes_emit(1, 2, 2, 2, 1, _lib.DTYPE_U8, kw.get("grid", p), *strides,
                                                           0.5, kw.get("cases", p), kw.get("scan", p),
                                                           kw.get("verts", p), kw.get("faces", p), None)
    for kw in ("grid", "cases", "scan", "verts", "faces"):
        assert emit(**{kw: None}) == _lib.EINVAL, kw
    back = lambda pad=1, **kw: lib.dibr_b200_marching_cubes_backward(1, 2, 2, 2, pad, kw.get("grid", p), *strides, 0.5,
                                                                      kw.get("cases", p), kw.get("scan", p),
                                                                      kw.get("grad", p), kw.get("out", p), None)
    assert back(pad=0) == _lib.EINVAL
    for kw in ("grid", "cases", "scan", "grad", "out"):
        assert back(**{kw: None}) == _lib.EINVAL, kw
    assert lib.dibr_b200_marching_cubes_case_table(None) == _lib.EINVAL
