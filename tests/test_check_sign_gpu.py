"""check_sign, CheckSign and _C.ops.mesh.unbatched_mesh_intersection_cuda (kaolin_b200/csrc/check_sign.cu)
against the reference's own CUDA operator (oracle/build_ref_check_sign.py), through its stored counts
(tests/golden/ref_cuda_check_sign.npz, oracle/ref_golden_check_sign.py), and against the brute-force C
oracle (oracle/check_sign.c), in float32 and float64.

The scenes (oracle/check_sign.py) are constructed around the places the binning could drop a pair or
the predicate could round differently: shared vertices and edges of lattices (edges of constant y take
the vertical-edge rule), points and face boxes on cell borders, faces of exactly the cell cap and more,
a mesh of wide faces only, G = 8 .. 256, three views with different vertices, NaN / inf / huge
coordinates, maxlen = 0 or set by an unreferenced vertex, duplicate faces.  tests/test_check_sign_cpu.py
shows with a host restatement of the binning that each scene reaches what it was built for."""
import warnings

import numpy as np
import pytest
import torch

from oracle import build_ref_check_sign, ref_golden_check_sign
from oracle import check_sign as oracle
from kaolin_b200 import _C, _lib
from kaolin_b200.ops.mesh import CheckSign, check_sign

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = {"f32": np.float32, "f64": np.float64}
SCENES = oracle.scenes()
MESH_SCENES = [n for n, s in SCENES.items() if not oracle.is_raw(s)]
RAW_SCENES = [n for n, s in SCENES.items() if oracle.is_raw(s)]


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _reference_counts(scene):
    """The reference's check_sign.py:138-155 up to the parity, on its operator (recording only)."""
    ref = build_ref_check_sign.load()
    assert ref is not None, "oracle/_ref/kaolin_ref_check_sign_C.so is not built"
    if oracle.is_raw(scene):
        return ref.unbatched_mesh_intersection_cuda(*(t(scene[k]) for k in ("points", "verts_1", "verts_2",
                                                                            "verts_3")))
    verts, faces, points = t(scene["verts"]), t(scene["faces"]), t(scene["points"])
    lens = [verts[..., a].max(-1)[0] - verts[..., a].min(-1)[0] for a in range(3)]
    maxlen = torch.max(torch.stack(lens), 0)[0]
    verts, points = verts / maxlen.view(-1, 1, 1), points / maxlen.view(-1, 1, 1)
    out = []
    for b in range(verts.shape[0]):
        v = [torch.index_select(verts[b], 0, faces[:, k]).contiguous() for k in range(3)]
        out.append(ref.unbatched_mesh_intersection_cuda(points[b].contiguous(), *v))
    return torch.stack(out)


def reference(name, dt):
    scene = oracle.cast(SCENES[name], DTYPES[dt])
    return ref_golden_check_sign.reference(f"{name}.{dt}", lambda: {"counts": _reference_counts(scene)},
                                           ("counts",), full=("counts",))


def _our_counts_via_C(scene):
    """check_sign.py's wrapper restated on this library's _C.ops.mesh operator."""
    verts, faces, points = t(scene["verts"]), t(scene["faces"]), t(scene["points"])
    lens = [verts[..., a].max(-1)[0] - verts[..., a].min(-1)[0] for a in range(3)]
    maxlen = torch.max(torch.stack(lens), 0)[0]
    verts, points = verts / maxlen.view(-1, 1, 1), points / maxlen.view(-1, 1, 1)
    out = []
    for b in range(verts.shape[0]):
        v = [torch.index_select(verts[b], 0, faces[:, k]).contiguous() for k in range(3)]
        out.append(_C.ops.mesh.unbatched_mesh_intersection_cuda(points[b].contiguous(), *v))
    return torch.stack(out)


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("name", MESH_SCENES)
def test_check_sign_equals_reference(name, dt):
    scene = oracle.cast(SCENES[name], DTYPES[dt])
    ref = reference(name, dt)
    ours = check_sign(t(scene["verts"]), t(scene["faces"]), t(scene["points"]))
    assert ours.dtype == torch.bool and tuple(ours.shape) == scene["points"].shape[:2]
    counts = ref.pair("counts", np.zeros(tuple(ours.shape), DTYPES[dt]))[1].reshape(tuple(ours.shape))
    np.testing.assert_array_equal(ours.cpu().numpy(), counts % 2 == 1)
    np.testing.assert_array_equal(ours.cpu().numpy(), oracle.check_sign(scene["verts"], scene["faces"],
                                                                        scene["points"]))
    # the reference's wrapper on this library's operator: the counts themselves, bit for bit
    assert ref.equal("counts", _our_counts_via_C(scene)), name


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("name", RAW_SCENES)
def test_raw_operator_equals_reference(name, dt):
    scene = oracle.cast(SCENES[name], DTYPES[dt])
    ref = reference(name, dt)
    ours = _C.ops.mesh.unbatched_mesh_intersection_cuda(*(t(scene[k]) for k in ("points", "verts_1", "verts_2",
                                                                                "verts_3")))
    assert ours.dtype == (torch.float32 if dt == "f32" else torch.float64)
    assert ref.equal("counts", ours), name
    np.testing.assert_array_equal(ours.cpu().numpy(), oracle.oracle_counts(scene))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_reference_fixture(dtype):
    """The reference test's meshes (B = 2), with and without its zero-area faces."""
    with np.load(oracle.FIXTURE) as z:
        verts, faces, points, expected = (t(z[k]) for k in ("verts", "faces", "points", "expected"))
        zero = t(z["zero_area_faces"])
    verts, points = verts.to(dtype), points.to(dtype)
    assert torch.equal(check_sign(verts[:1], faces, points[:1]), expected[:1])
    assert torch.equal(check_sign(verts, faces, points), expected)
    assert torch.equal(check_sign(verts, torch.cat([faces, zero]), points), expected)
    S = CheckSign(verts, faces)
    assert torch.equal(S(points), expected)


def _noisy_icosphere(level, seed):
    """Radial noise of a fifth of the edge length (about 1 / 2^level)."""
    rng = np.random.default_rng(seed)
    v, f = oracle._icosphere(level, rng, 0.2 / 2 ** level)
    return v, f, rng


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_icosphere_million_points_against_oracle(dtype):
    """Level 6 (81 920 faces) with noise, 10^6 uniform points in its box; the C oracle on a sample."""
    v, f, rng = _noisy_icosphere(6, 6)
    v = v.astype(dtype)
    q = oracle._uniform(rng, v.astype(np.float64), 1_000_000, 0.05).astype(dtype)
    ours = check_sign(t(v[None]), t(f), t(q[None]))[0].cpu().numpy()
    inside = np.linalg.norm(q, axis=1) < 0.94
    outside = np.linalg.norm(q, axis=1) > 1.06
    assert ours[inside].all() and not ours[outside].any()
    pick = np.sort(rng.choice(len(q), 3000, replace=False))
    np.testing.assert_array_equal(ours[pick], oracle.check_sign(v[None], f, q[pick][None])[0])


def test_reruns_are_byte_identical():
    s = SCENES["batch3"]
    verts, faces, points = t(s["verts"]), t(s["faces"]), t(s["points"])
    a = check_sign(verts, faces, points)
    S = CheckSign(verts, faces)
    assert torch.equal(a, S(points)) and torch.equal(a, S(points)) and torch.equal(a, check_sign(verts, faces, points))
    raw = SCENES["raw_soup"]
    args = [t(raw[k]) for k in ("points", "verts_1", "verts_2", "verts_3")]
    c0, c1 = (_C.ops.mesh.unbatched_mesh_intersection_cuda(*args) for _ in range(2))
    assert torch.equal(c0, c1)


def test_one_sync_per_build_none_per_query():
    s = SCENES["batch3"]
    verts, faces, points = t(s["verts"]), t(s["faces"]), t(s["points"])
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as got:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            S = CheckSign(verts, faces)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    syncs = [w for w in got if "called a synchronizing" in str(w.message)]
    assert len(syncs) == 1, [str(w.message) for w in got]
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = S(points)
        out2 = S(points * 0.5)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(out, check_sign(verts, faces, points))
    assert torch.equal(out2, check_sign(verts, faces, points * 0.5))


def test_peak_memory_within_layout_bound():
    """Level 7 (327 680 faces), B = 2, 2 * 10^6 points: the call allocates the build and query
    workspaces and the output, nothing else."""
    v, f, rng = _noisy_icosphere(7, 7)
    B, N = 2, 2_000_000
    verts = t(np.stack([v, v * 1.5]).astype(np.float32))
    faces = t(f)
    points = t(np.stack([oracle._uniform(rng, v, N, 0.0), oracle._uniform(rng, v * 1.5, N, 0.0)]).astype(np.float32))
    build, query = _lib.check_sign_workspace_bytes(B, f.shape[0], N, _lib.DTYPE_F32, "test")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = check_sign(verts, faces, points)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    # four allocations: build and query workspaces, the output and the status word; the caching
    # allocator may hand out up to 2 MiB more than asked for a large block it does not split
    bound = build + query + B * N + 512 + 3 * (2 << 20)
    assert peak <= bound, (peak, bound)
    # layout: B*F*16 entries, B*F wide ids, boxes, 9 coordinates, per point a cell and an order slot
    F = f.shape[0]
    assert build < B * F * (16 * 4 + 4 + 16 + 9 * 4) + 4 * B * (256 * 256 + 1) * 4 + 4096
    assert query < 2 * B * N * 4 + 2 * B * (256 * 256 + 1) * 4 + 2048
    assert 0.45 < out.float().mean().item() < 0.6        # a ball fills pi / 6 of its box


def test_deviations():
    s = oracle.cast(SCENES["batch3"], np.float32)
    verts, faces, points = t(s["verts"]), t(s["faces"]), t(s["points"])
    # F = 0: every point outside (the reference's launch of zero blocks fails)
    empty = torch.zeros((0, 3), dtype=torch.int64, device=DEV)
    out = check_sign(verts, empty, points)
    assert out.shape == points.shape[:2] and not out.any()
    assert torch.equal(CheckSign(verts, empty)(points), out)
    assert not _C.ops.mesh.unbatched_mesh_intersection_cuda(points[0], *(points.new_zeros((0, 3)),) * 3).any()
    # B = 0: a (0, N) tensor (the reference's torch.stack([]) raises)
    out = check_sign(verts[:0], faces, points[:0])
    assert out.shape == (0, points.shape[1]) and out.dtype == torch.bool
    # an index outside [0, V): IndexError (the reference's index_select faults on the device)
    V = verts.shape[1]
    for bad in (V, -1):
        f = faces.clone()
        f[5, 1] = bad
        with pytest.raises(IndexError):
            check_sign(verts, f, points)
        with pytest.raises(IndexError):
            CheckSign(verts, f)
    # no CPU path, and verts and points of one float type
    with pytest.raises(RuntimeError):
        check_sign(verts.cpu(), faces.cpu(), points.cpu())
    with pytest.raises(RuntimeError):
        check_sign(verts, faces, points.double())
    with pytest.raises(RuntimeError):
        check_sign(verts.half(), faces, points.half())
    # hash_resolution is checked and otherwise unused
    assert torch.equal(check_sign(verts, faces, points, 7), check_sign(verts, faces, points))


def test_raw_operator_argument_checks():
    p = torch.zeros((4, 3), device=DEV)
    v = torch.zeros((2, 3), device=DEV)
    op = _C.ops.mesh.unbatched_mesh_intersection_cuda
    with pytest.raises(RuntimeError):
        op(p.double(), v.double(), v.double(), v)                      # checkAllSameType
    with pytest.raises(RuntimeError):
        op(p, v, v, torch.zeros((3, 3), device=DEV))                   # checkSize
    with pytest.raises(RuntimeError):
        op(p[:, :2].contiguous(), v, v, v)
    with pytest.raises(RuntimeError):
        op(p.t().contiguous().t(), v, v, v)                            # checkAllContiguous
    with pytest.raises(RuntimeError):
        op(p.half(), v.half(), v.half(), v.half())                     # dispatch: float and double only
    assert op(p, v, v, v).dtype == torch.float32 and not op(p, v, v, v).any()


def test_workspace_at_an_odd_address(monkeypatch):
    """Every workspace starting at byte 1 of a larger buffer: the outputs of an aligned one."""
    s = SCENES["batch3"]
    verts, faces, points = t(s["verts"]), t(s["faces"]), t(s["points"])
    raw = SCENES["raw_soup"]
    args = [t(raw[k]) for k in ("points", "verts_1", "verts_2", "verts_3")]

    def run():
        return [check_sign(verts, faces, points), CheckSign(verts, faces)(points),
                _C.ops.mesh.unbatched_mesh_intersection_cuda(*args)]

    want = run()
    scratch, odd = _lib.scratch, []
    monkeypatch.setattr(_lib, "scratch", lambda n, device: odd.append(n) or scratch(int(n) + 1, device)[1:])
    got = run()
    assert odd
    for a, b in zip(want, got):
        assert torch.equal(a, b)
