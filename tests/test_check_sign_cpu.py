"""check_sign without a GPU: the C oracle (oracle/check_sign.c) against the reference's test fixture and
the reference operator's stored counts, the reference's argument errors, the host-side errors of the
C ABI, and a host restatement of the binning showing each constructed scene reaches what it was built for."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import check_sign as oracle
from oracle import ref_golden_check_sign
from kaolin_b200 import _lib
from kaolin_b200.ops.mesh import CheckSign, check_sign

SCENES = oracle.scenes()


@pytest.mark.parametrize("zero_area", [False, True])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_oracle_reproduces_reference_test(dtype, zero_area):
    with np.load(oracle.FIXTURE) as z:
        faces = np.concatenate([z["faces"], z["zero_area_faces"]]) if zero_area else z["faces"]
        out = oracle.check_sign(z["verts"].astype(dtype), faces, z["points"].astype(dtype))
        np.testing.assert_array_equal(out, z["expected"])
        np.testing.assert_array_equal(oracle.check_sign(z["verts"][:1].astype(dtype), faces,
                                                        z["points"][:1].astype(dtype)), z["expected"][:1])


def _stored_cases():
    return sorted(ref_golden_check_sign._load())


def test_every_scene_has_stored_reference_counts():
    expected = {f"{n}p{dt}" for n in SCENES for dt in ("f32", "f64")}     # the store writes "." as "p"
    assert set(_stored_cases()) == expected


@pytest.mark.parametrize("case", _stored_cases())
def test_oracle_reproduces_stored_reference_counts(case):
    name, dt = case.rsplit("p", 1)
    scene = oracle.cast(SCENES[name], {"f32": np.float32, "f64": np.float64}[dt])
    ref = ref_golden_check_sign.reference(case, None, ("counts",))
    ours = oracle.oracle_counts(scene)
    assert ref.equal("counts", ours), case


# ---- the scenes reach the borders they were built for (host restatement of the binning) ----

def _on_border(c, G):
    return int((np.isfinite(c) & (c == np.floor(c)) & (c >= 1) & (c <= G - 1)).sum())


def _views(name):
    return oracle.binning(SCENES[name])


@pytest.mark.parametrize("name", ["lattice", "cell_borders_cap"])
def test_points_and_boxes_on_cell_borders(name):
    for v in _views(name):
        assert _on_border(v["point_coord"][0], v["G"]) + _on_border(v["point_coord"][1], v["G"]) > 1000
        assert _on_border(v["box_coord"][0], v["G"]) + _on_border(v["box_coord"][1], v["G"]) > 500


def test_cap_and_wide_faces():
    (v,) = _views("cell_borders_cap")
    assert v["G"] == 32
    assert (v["ncell"] == oracle.CAP).sum() >= 12 and (v["ncell"] == oracle.CAP + 1).sum() >= 4
    (w,) = _views("wide_only")
    assert (w["ncell"] > oracle.CAP).all()


def test_grid_sides_span_the_range():
    got = {v["G"] for n in SCENES if n.startswith("soup_") for v in _views(n)}
    assert {8, 256} <= got and len(got) == 4
    assert {v["G"] for v in _views("batch3")} == {40} and len(_views("batch3")) == 3


def test_lattice_points_on_shared_vertices_and_vertical_edges():
    s = SCENES["lattice"]
    v = s["verts"][0]
    yz = {tuple(r) for r in v[:, 1:]}
    pts = s["points"][0]
    on_vertex = np.array([tuple(r) in yz for r in pts[:, 1:]])
    assert on_vertex.sum() >= 81 * 6
    # edges of constant y (the reference's "completely vertical" 2-D edge): y on the lattice, z between
    on_y = np.isin(pts[:, 1], v[:, 1]) & ~np.isin(pts[:, 2], v[:, 2])
    assert on_y.sum() >= 72 * 6


def test_degenerate_scenes_reach_their_cases():
    (d,) = _views("raw_nan_inf")
    assert (d["ncell"] == 0).sum() == 100                # all-NaN y or z boxes: dropped
    (f,) = _views("far_points")
    c = f["point_coord"][0]
    assert (c < 0).sum() > 50 and (c > f["G"]).sum() > 50  # clamped to the border cells
    pts = SCENES["nan_inf_points"]["points"][0]
    assert np.isnan(pts).any() and np.isinf(pts).any()
    v = SCENES["zero_maxlen"]["verts"][0]
    assert (np.ptp(v, axis=0) == 0).all()
    far = SCENES["far_vertex"]
    assert far["verts"][0, -1, 0] == 1e6 and far["faces"].max() < far["verts"].shape[1] - 1


# ---- the reference's argument errors, in its order (check_sign.py:104-136; test_check_sign.py) ----

def _fixture():
    with np.load(oracle.FIXTURE) as z:
        return torch.from_numpy(z["verts"]).float(), torch.from_numpy(z["faces"]), torch.from_numpy(z["points"]).float()


@pytest.mark.parametrize("mutate, exc, msg", [
    (lambda v, f, p, h: (v, f.int(), p, h), TypeError, r"Expected faces entries to be torch.int64 but got torch.int32."),
    (lambda v, f, p, h: (v, f, p, 512.0), TypeError,
     r"Expected hash_resolution to be int but got <class 'float'>."),
    (lambda v, f, p, h: (v.unsqueeze(-1), f, p, h), ValueError, r"Expected verts to have 3 dimensions but got 4 dimensions."),
    (lambda v, f, p, h: (v, f.unsqueeze(-1), p, h), ValueError, r"Expected faces to have 2 dimensions but got 3 dimensions."),
    (lambda v, f, p, h: (v, f, p.unsqueeze(-1), h), ValueError,
     r"Expected points to have 3 dimensions but got 4 dimensions."),
    (lambda v, f, p, h: (v[..., :2], f, p, h), ValueError, r"Expected verts to have 3 coordinates but got 2 coordinates."),
    (lambda v, f, p, h: (v, f[:, :2], p, h), ValueError, r"Expected faces to have 3 vertices but got 2 vertices."),
    (lambda v, f, p, h: (v, f, p[..., :2], h), ValueError,
     r"Expected points to have 3 coordinates but got 2 coordinates."),
    # two errors at once: the reference's order decides which is raised
    (lambda v, f, p, h: (v.unsqueeze(-1), f.int(), p, 1.5), TypeError, r"Expected faces entries to be torch.int64"),
    (lambda v, f, p, h: (v[..., :2], f.unsqueeze(-1), p, h), ValueError, r"Expected faces to have 2 dimensions"),
])
def test_argument_errors_match_the_reference(mutate, exc, msg):
    v, f, p, h = mutate(*_fixture(), 512)
    with pytest.raises(exc, match=msg):
        check_sign(v, f, p, h)


def test_cpu_tensors_have_no_path():
    v, f, p = _fixture()
    with pytest.raises(RuntimeError, match="CUDA"):
        check_sign(v, f, p)
    with pytest.raises(RuntimeError, match="CUDA"):
        CheckSign(v, f)


# ---- host-side errors of the C ABI (fake pointers; nothing reaches the device) ----

FAKE = ctypes.c_void_p(0x100000)


def test_abi_workspace_bytes_errors():
    L = _lib.lib()
    b, q = ctypes.c_size_t(0), ctypes.c_size_t(0)
    assert L.dibr_b200_check_sign_workspace_bytes(1, 10, 10, 2, ctypes.byref(b), ctypes.byref(q)) == _lib.EINVAL
    assert L.dibr_b200_check_sign_workspace_bytes(0, 10, 10, 0, ctypes.byref(b), ctypes.byref(q)) == _lib.EINVAL
    assert L.dibr_b200_check_sign_workspace_bytes(1, -1, 10, 0, ctypes.byref(b), ctypes.byref(q)) == _lib.EINVAL
    assert L.dibr_b200_check_sign_workspace_bytes(1, 10, -1, 1, ctypes.byref(b), ctypes.byref(q)) == _lib.EINVAL
    assert L.dibr_b200_check_sign_workspace_bytes(8, 1 << 24, 10, 0, ctypes.byref(b), ctypes.byref(q)) == _lib.ESIZE
    assert L.dibr_b200_check_sign_workspace_bytes(2, 10, 1 << 30, 0, ctypes.byref(b), ctypes.byref(q)) == _lib.ESIZE
    assert L.dibr_b200_check_sign_workspace_bytes(2, 1000, 500, 1, ctypes.byref(b), ctypes.byref(q)) == 0
    b32 = _lib.check_sign_workspace_bytes(2, 1000, 500, _lib.DTYPE_F32, "t")
    assert b.value > b32[0] and q.value == b32[1]      # float64 records are wider; the query is type-free


def test_abi_build_and_query_errors():
    L = _lib.lib()
    build, query = _lib.check_sign_workspace_bytes(2, 100, 50, _lib.DTYPE_F32, "t")
    args = lambda **kw: [kw.get(k, d) for k, d in (("B", 2), ("V", 60), ("F", 100), ("dt", 0), ("verts", FAKE),
                                                     ("faces", FAKE), ("status", FAKE), ("ws", FAKE),
                                                     ("bytes", build), ("stream", None))]
    assert L.dibr_b200_check_sign_build(*args(dt=5)) == _lib.EINVAL
    assert L.dibr_b200_check_sign_build(*args(B=0)) == _lib.EINVAL
    assert L.dibr_b200_check_sign_build(*args(F=-1)) == _lib.EINVAL
    assert L.dibr_b200_check_sign_build(*args(faces=None)) == _lib.EINVAL
    assert L.dibr_b200_check_sign_build(*args(status=None)) == _lib.EINVAL
    assert L.dibr_b200_check_sign_build(*args(F=1 << 28)) == _lib.ESIZE
    assert L.dibr_b200_check_sign_build(*args(bytes=build - 1)) == _lib.EWORKSPACE
    q = lambda **kw: [kw.get(k, d) for k, d in (("B", 2), ("F", 100), ("N", 50), ("dt", 0), ("points", FAKE),
                                                  ("mesh", FAKE), ("mesh_bytes", build), ("inside", FAKE),
                                                  ("ws", FAKE), ("bytes", query), ("stream", None))]
    assert L.dibr_b200_check_sign_query(*q(dt=-1)) == _lib.EINVAL
    assert L.dibr_b200_check_sign_query(*q(inside=None)) == _lib.EINVAL
    assert L.dibr_b200_check_sign_query(*q(N=1 << 30)) == _lib.ESIZE
    assert L.dibr_b200_check_sign_query(*q(mesh_bytes=build - 1)) == _lib.EWORKSPACE
    assert L.dibr_b200_check_sign_query(*q(bytes=query - 1)) == _lib.EWORKSPACE
    b1, q1 = _lib.check_sign_workspace_bytes(1, 100, 50, _lib.DTYPE_F64, "t")
    r = lambda **kw: [kw.get(k, d) for k, d in (("F", 100), ("N", 50), ("dt", 1), ("points", FAKE), ("v1", FAKE),
                                                  ("v2", FAKE), ("v3", FAKE), ("counts", FAKE), ("ws", FAKE),
                                                  ("bytes", b1 + q1), ("stream", None))]
    assert L.dibr_b200_mesh_intersection_count(*r(dt=3)) == _lib.EINVAL
    assert L.dibr_b200_mesh_intersection_count(*r(v2=None)) == _lib.EINVAL
    assert L.dibr_b200_mesh_intersection_count(*r(counts=None)) == _lib.EINVAL
    assert L.dibr_b200_mesh_intersection_count(*r(F=1 << 28)) == _lib.ESIZE
    assert L.dibr_b200_mesh_intersection_count(*r(bytes=b1 + q1 - 1)) == _lib.EWORKSPACE


def test_golden_fixture_is_the_reference_tests():
    with np.load(oracle.FIXTURE) as z:
        assert z["verts"].shape == (2, 8, 3) and z["faces"].shape == (12, 3) and z["points"].shape == (2, 33, 3)
        assert z["expected"][0, :10].all() and not z["expected"][0, 10:].any()
        np.testing.assert_array_equal(z["verts"][1], -z["verts"][0])
    assert os.path.getsize(oracle.FIXTURE) < 4096
