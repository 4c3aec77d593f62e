"""CPU checks of surface sampling: the numpy oracle's Philox against the Random123 known answers, the
oracle against the reference's stored outputs (tests/golden/sample_points.npz) bit for bit, the
distribution the random-stream contract gives, the workspace layout and the C ABI's host-side limits."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
from scipy import stats

from kaolin_b200 import _lib, synthetic
from oracle import sample_points as osp

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "sample_points.npz")
SRC = os.path.join(ROOT, "tests", "host_math", "sample_points_layout.cpp")
HDR = os.path.join(ROOT, "kaolin_b200", "csrc", "op_layouts.h")
LIB = os.path.join(ROOT, "tests", "host_math", "_build", "sample_points_layout.so")
ALIGN = 256
INT32_MAX = 2 ** 31 - 1


def _stored():
    z = np.load(GOLDEN)
    out = {}
    for k in z.files:
        scene, dt, name = k.split("/")
        x = z[k]
        out.setdefault((scene, dt), {})[name] = x.astype(np.int64) if x.dtype.kind == "i" else x
    return out


STORED = _stored()
DENSE = sorted(k for k, r in STORED.items() if "first_idx" not in r)
PACKED = sorted(k for k, r in STORED.items() if "first_idx" in r)


# Random123 (Salmon et al., SC 2011) known answers of Philox4x32-10.
@pytest.mark.parametrize("counter,key,expect", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(counter, key, expect):
    assert tuple(int(w) for w in osp.philox(*counter, *key)) == expect


def test_uniform_maps():
    r, u, v = osp.uniforms(123, 3, 1000, np.float32)
    assert r.dtype == np.float64 and u.dtype == np.float32 and v.dtype == np.float32
    assert (r >= 0).all() and (r < 1).all() and (u >= 0).all() and (u < 1).all()
    assert np.array_equal(r * 2.0 ** 53, np.floor(r * 2.0 ** 53))
    assert np.array_equal(u * 2.0 ** 24, np.floor(u * 2.0 ** 24))
    r64, u64, v64 = osp.uniforms(123, 3, 1000, np.float64)
    assert np.array_equal(r, r64)               # block 0, words 0 and 1 in both dtypes
    assert np.array_equal(u64 * 2.0 ** 53, np.floor(u64 * 2.0 ** 53)) and not np.array_equal(u64, v64)
    assert not np.array_equal(osp.uniforms(124, 3, 1000, np.float32)[0], r)
    assert osp.key_halves(-1) == (0xFFFFFFFF, 0xFFFFFFFF) and osp.key_halves(1 << 32) == (0, 1)


def test_choice_rules():
    c = np.array([0.0, 1.0, 1.0, 3.0, 3.0])   # faces 0, 2 and 4 have zero area
    f, _ = osp.choose(c, np.array([0.0, 0.2, 1 / 3, 0.5, 0.999999]))
    assert f.tolist() == [1, 1, 3, 3, 3]
    f, _ = osp.choose(c, np.array([np.nextafter(1.0, 0.0)]))
    assert f.tolist() == [3]


@pytest.mark.parametrize("scene,dt", DENSE)
def test_oracle_equals_stored_reference(scene, dt):
    r = STORED[(scene, dt)]
    given = r.get("given_areas")
    ff = r.get("face_features")
    pts, ch, feats, _, _ = osp.sample_points(r["vertices"], r["faces"], int(r["N"]), int(r["key"]), areas=given,
                                             face_features=ff)
    assert np.array_equal(osp.face_areas(r["vertices"], r["faces"]), r["areas"])
    assert np.array_equal(ch, r["choices"])
    assert np.array_equal(pts, r["points"])
    if ff is not None:
        assert np.array_equal(feats, r["features"])


@pytest.mark.parametrize("scene,dt", PACKED)
def test_oracle_equals_stored_packed_reference(scene, dt):
    r = STORED[(scene, dt)]
    nfm, first = r["num_faces"], r["first_idx"]
    merged = r["faces"] + np.repeat(first[:-1], nfm)[:, None]
    off = np.concatenate([[0], np.cumsum(nfm)])
    areas = osp.face_areas(r["vertices"][None], merged)[0]
    assert np.array_equal(areas, r["areas"])
    B, N = nfm.shape[0], int(r["N"])
    rr, u, v = osp.uniforms(int(r["key"]), B, N, r["vertices"].dtype)
    for b in range(B):
        f, _ = osp.choose(osp.cdf(areas[off[b]:off[b + 1]]), rr[b])
        assert np.array_equal(f + off[b], r["choices"][b])
    w = osp.weights(u, v)
    pts = osp.interpolate(w, *(r["vertices"][merged[r["choices"], k]] for k in range(3)))
    assert np.array_equal(pts, r["points"])


@pytest.mark.parametrize("scene,dt", DENSE)
def test_oracle_gradients_match_stored_reference(scene, dt):
    r = STORED[(scene, dt)]
    _, u, v = osp.uniforms(int(r["key"]), r["vertices"].shape[0], int(r["N"]), r["vertices"].dtype)
    ff = r.get("face_features")
    gv, gf = osp.grad_sample_points(r["vertices"].shape, r["faces"], r["choices"], osp.weights(u, v),
                                    r["grad_points"], None if ff is None else ff.shape, r.get("grad_features"))
    tol = 1e-6 if dt == "f32" else 1e-12
    scale = max(np.abs(gv).max(), 1.0)
    assert np.abs(gv - r["ref_grad_vertices"]).max() <= tol * scale
    if ff is not None:
        assert np.abs(gf - r["ref_grad_face_features"]).max() <= tol * max(np.abs(gf).max(), 1.0)
    ga = osp.grad_face_areas(r["vertices"], r["faces"], r["grad_areas"])
    ref = r["ref_grad_vertices_areas"]
    assert np.array_equal(np.isnan(ga), np.isnan(ref))
    ok = ~np.isnan(ref)
    assert np.abs(ga[ok] - ref[ok]).max() <= 1e-4 * max(np.abs(ga[ok]).max(), 1.0)


def test_degenerate_scene_has_nan_area_gradients():
    for dt in ("f32", "f64"):
        r = STORED[("degenerate", dt)]
        assert (r["areas"] == 0).any()
        assert np.isnan(r["ref_grad_vertices_areas"]).any()
        zero = np.flatnonzero(r["areas"][0] == 0)
        assert not np.isin(r["choices"], zero).any()       # a zero-area face is never chosen


def test_given_areas_scene_skips_zero_faces():
    r = STORED[("given_areas", "f32")]
    for b in range(2):
        assert (r["given_areas"][b][r["choices"][b]] > 0).all()


def _uneven_mesh():
    v, f = synthetic.icosphere(2)
    v = np.asarray(v, np.float64)
    v = v * (1.0 + 0.6 * v[:, :1] ** 2)          # stretch: face areas vary by about 4x
    return v[None], np.asarray(f, np.int64)


def test_face_choice_distribution_chi_square():
    v, f = _uneven_mesh()
    N = 10 ** 6
    areas = osp.face_areas(v, f)[0]
    r, _, _ = osp.uniforms(0x5EED, 1, N, np.float64)
    ch, _ = osp.choose(osp.cdf(areas), r[0])
    counts = np.bincount(ch, minlength=f.shape[0])
    expect = N * areas / areas.sum()
    p = stats.chisquare(counts, expect).pvalue
    assert p > 1e-4, p


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_barycentrics_uniform_on_the_triangle(dtype):
    # uniform on a triangle: w2 / (w1 + w2) = v ~ U(0, 1) and w1 + w2 = sqrt(u_raw) has density 2x
    _, u, v = osp.uniforms(0xC0FFEE, 1, 10 ** 6, dtype)
    w0, w1, w2 = osp.weights(u[0], v[0])
    s = np.asarray(w1, np.float64) + np.asarray(w2, np.float64)
    assert stats.kstest(s, lambda x: np.clip(x, 0, 1) ** 2).pvalue > 1e-4
    ok = s > 0
    assert stats.kstest(np.asarray(w2, np.float64)[ok] / s[ok], "uniform").pvalue > 1e-4
    assert np.abs(np.asarray(w0, np.float64) + s - 1).max() <= 4 * np.finfo(dtype).eps


# ---------------------------------------------------------------------------------------------
# Workspace layout and the C ABI's host-side checks.

@pytest.fixture(scope="module")
def sp():
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(SRC), os.path.getmtime(HDR)):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", LIB, SRC])
    lib = ctypes.CDLL(LIB)
    lib.sp_layout.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int64,
                              ctypes.POINTER(ctypes.c_int64)]
    lib.sp_carve.argtypes = [ctypes.c_uint64] * 3
    lib.sp_carve.restype = ctypes.c_int64
    return lib


FWD = ("cdf", "coarse", "tile_sum", "tile_flag", "carry", "view_flag")
BWD = ("corner_grad", "count", "off", "sums", "ids", "long_rows", "long_count")
SHAPES = [(1, 1, 0), (1, 1, 1), (2, 2560, 1500), (8, 8 * 81920, 100000), (1, 4096, 4097), (1, 4097, 1),
          (1, 16785218, 50000), (3, 700_000_000, 1), (1, 1, INT32_MAX - 1)]


def needs(backward, B, nf, N, ts):
    """Bytes each piece's kernels index."""
    tiles = (nf + 4095) // 4096
    if not backward:
        return {"cdf": nf * 8, "coarse": tiles * 8, "tile_sum": tiles * 8, "tile_flag": tiles * 4,
                "carry": tiles * 8, "view_flag": B * 4}
    return {"corner_grad": nf * 9 * ts, "count": nf * 4, "off": (nf + 1) * 4, "sums": 4 * ((nf + 4095) // 4096 + 1),
            "ids": B * N * 4, "long_rows": nf * 4, "long_count": 4}


@pytest.mark.parametrize("backward", [0, 1])
def test_layout_pieces_are_aligned_apart_and_inside(sp, backward):
    names = BWD if backward else FWD
    for B, nf, N in SHAPES:
        for ts in (4, 8):
            out = (ctypes.c_int64 * 32)()
            assert sp.sp_layout(backward, B, nf, N, ts, out) == 1 + 2 * len(names)
            total = out[0]
            pieces = {n: (out[1 + 2 * i], out[2 + 2 * i]) for i, n in enumerate(names)}
            for name, need in needs(backward, B, nf, N, ts).items():
                assert pieces[name][1] >= need, (B, nf, N, ts, name)
            spans = sorted((at, at + n) for at, n in pieces.values() if n > 0)
            for (_, e0), (s1, _) in zip(spans, spans[1:]):
                assert e0 <= s1
            for offset in (0, 1, 3, 8, 255):
                ws = 0x10000 + offset
                origin = sp.sp_carve(ws, total, total)
                assert 0 <= origin < ALIGN and (ws + origin) % ALIGN == 0
                for at, n in pieces.values():
                    assert (ws + origin + at) % ALIGN == 0 and origin + at + n <= total
                assert sp.sp_carve(ws, total - 1, total) == -1


def test_size_query_returns_the_layout_totals(sp):
    for B, nf, N in [(1, 1, 1), (2, 2560, 1500), (3, 1000, 0), (8, 655360, 100000)]:
        for dtype, ts in ((_lib.DTYPE_F32, 4), (_lib.DTYPE_F64, 8)):
            fwd, bwd = _lib.sample_points_workspace_bytes(B, nf, N, dtype, "q")
            for backward, got in ((0, fwd), (1, bwd)):
                out = (ctypes.c_int64 * 32)()
                sp.sp_layout(backward, B, nf, N, ts, out)
                assert got == out[0]


def test_c_abi_size_limits_and_arguments():
    lib = _lib.lib()
    f, b = ctypes.c_size_t(0), ctypes.c_size_t(0)
    q = lib.dibr_b200_sample_points_workspace_bytes
    assert q(1, INT32_MAX // 3 + 1, 1, _lib.DTYPE_F32, ctypes.byref(f), ctypes.byref(b)) == _lib.ESIZE
    assert q(1, INT32_MAX // 3 - 1, 1, _lib.DTYPE_F32, ctypes.byref(f), ctypes.byref(b)) == 0
    assert q(2, 10, 2 ** 30, _lib.DTYPE_F64, ctypes.byref(f), ctypes.byref(b)) == _lib.ESIZE
    assert q(1, 10, 1, 7, ctypes.byref(f), ctypes.byref(b)) == _lib.EINVAL
    assert q(-1, 10, 1, _lib.DTYPE_F32, ctypes.byref(f), ctypes.byref(b)) == _lib.EINVAL
    # NULL buffers are rejected on the host, before any launch
    assert lib.dibr_b200_sample_points_forward(1, 4, 3, 4, 3, _lib.DTYPE_F32, 10, 0, None, None, None, None, None,
                                               None, None, None, None, None, None, 0, None) == _lib.EINVAL
    assert lib.dibr_b200_sample_points_backward(1, 4, 3, 4, 3, _lib.DTYPE_F32, 10, 0, None, None, None, None, None,
                                                None, None, None, None, None, 0, None) == _lib.EINVAL
    assert lib.dibr_b200_face_areas_forward(1, 4, 3, 4, 3, _lib.DTYPE_F32, None, None, None, None, None,
                                            None) == _lib.EINVAL
    assert lib.dibr_b200_face_areas_backward(1, 4, 3, 4, 3, _lib.DTYPE_F32, None, None, None, None, None, None,
                                             None, None, 0, None) == _lib.EINVAL
