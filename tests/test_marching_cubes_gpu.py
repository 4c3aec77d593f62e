"""Marching cubes on sm_90a (csrc/marching_cubes.cu) against the reference's own CUDA operator
(tests/golden/ref_cuda_mcube.npz, recorded from oracle/_ref through the reference wrapper's per-view
steps) and the numpy restatement (oracle/marching_cubes.py): vertices and faces bit-equal to both,
all views batched in one call; each deliberate deviation against the corrected restatement, and
different from the reference's recorded wrong outputs; every
input dtype and non-contiguous input; byte-identical reruns; one synchronising read per call and
none in the backward; gradients against float64 autograd; 256^3 with two views in bounded memory."""
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from kaolin_b200 import _C, _lib
from kaolin_b200.ops import conversions
from oracle import build_ref_mcube, ref_golden_mcube
from oracle import marching_cubes as O
from oracle.marching_cubes import QUIRKS, SCENES, checker, occupancy, same_bits, sphere

pytestmark = pytest.mark.gpu
DEV = "cuda"
mc = conversions.voxelgrids_to_trianglemeshes


def ref_wrapper(voxelgrids, iso_value=0.5):
    """The reference's voxelgrids_to_trianglemeshes (voxelgrid.py:217-246), step for step, on the
    reference's operator built under oracle/_ref."""
    mod = build_ref_mcube.load()
    if mod is None:
        pytest.skip("oracle/_ref/kaolin_ref_mcube_C.so is not built")
    vg = F.pad(voxelgrids.float(), (1, 1, 1, 1, 1, 1), "constant", 0)
    verts, faces = [], []
    for i in range(vg.shape[0]):
        cur = vg[i]
        if torch.all(cur == 0):
            verts.append(torch.zeros((0, 3), dtype=torch.float, device=vg.device))
            faces.append(torch.zeros((0, 3), dtype=torch.long, device=vg.device))
            continue
        v, f = mod.unbatched_mcube_forward_cuda(cur, iso_value)
        verts.append(v)
        faces.append(f.long())
    return verts, faces


def reference(name, scenes=SCENES):
    make, iso = scenes[name]
    grid = make()
    B = grid.shape[0]

    def live():
        v, f = ref_wrapper(torch.from_numpy(grid).to(DEV), iso)
        out = {}
        for b in range(B):
            out[f"v{b}"], out[f"f{b}"] = v[b], f[b]
        return out
    names = [f"{k}{b}" for b in range(B) for k in "vf"]
    return grid, iso, ref_golden_mcube.reference(name, live, names, full=names if name == "cases" else ())


def oracle_table():
    _, _, ref = reference("cases")
    return O.Tables(O.case_table_from_golden(
        [(ref_golden_mcube.rows(ref, f"v{k}")[1], ref_golden_mcube.rows(ref, f"f{k}")[1]) for k in range(256)]))


_TABLES = []


def tables():
    if not _TABLES:
        _TABLES.append(oracle_table())
    return _TABLES[0]


def oracle(grid, iso, pad=1):
    return O.extract(grid, iso, tables(), pad)


def as_np(t):
    return t.detach().cpu().numpy()


@pytest.mark.parametrize("name", list(SCENES))
def test_equals_reference(name):
    grid, iso, ref = reference(name)
    verts, faces = mc(torch.from_numpy(grid).to(DEV), iso)
    assert len(verts) == len(faces) == grid.shape[0]
    for b in range(grid.shape[0]):
        assert ref.equal(f"v{b}", verts[b]), (name, b)
        assert ref.equal(f"f{b}", faces[b]), (name, b)


@pytest.mark.parametrize("name", ["specials", "iso_low", "views", "noisy32"])
def test_raw_operator_equals_reference(name):
    """The reference wrapper's steps on this library's _C operator."""
    grid, iso, ref = reference(name)
    vg = F.pad(torch.from_numpy(grid).to(DEV).float(), (1,) * 6)
    for b in range(grid.shape[0]):
        v, f = _C.ops.conversions.unbatched_mcube_forward_cuda(vg[b], iso)
        assert v.dtype == torch.float32 and f.dtype == torch.int32
        assert ref.equal(f"v{b}", v) and ref.equal(f"f{b}", f.long()), (name, b)


def test_case_table_from_reference_equals_library():
    ours = conversions.voxelgrid.case_table().numpy()
    for cs, edges in enumerate(tables().table):
        got = [O.EDGES.index(tuple(p)) if tuple(p) in O.EDGES else None for p in ours[cs].reshape(-1, 2) if p[0] >= 0]
        assert got == edges, cs


def check_against_oracle(grid, iso, verts, faces):
    for b in range(grid.shape[0]):
        ov, of, _ = oracle(grid[b].astype(np.float32), iso)
        assert same_bits(as_np(verts[b]), ov), b
        assert np.array_equal(as_np(faces[b]), of), b


ORACLE_SCENES = {
    "smooth32": lambda: (occupancy(32, 11)[None], 0.5),
    "noisy64": lambda: (np.random.default_rng(12).random((1, 64, 64, 64)).astype(np.float32), 0.3),
    "sphere128_u8": lambda: ((sphere(128) < 0.75).astype(np.uint8)[None], 0.5),
    "views3": lambda: (np.stack([occupancy(40, 13), (sphere(40) < 0.5).astype(np.float32),
                                 np.random.default_rng(14).random((40, 40, 40)).astype(np.float32)]), 0.5),
    "noncubic_37x64x50": lambda: (np.random.default_rng(15).random((1, 37, 64, 50)).astype(np.float32), 0.5),
    "noncubic_binary": lambda: ((np.random.default_rng(16).random((2, 9, 30, 17)) < 0.4).astype(np.float32), 0.5),
}


@pytest.mark.parametrize("name", list(ORACLE_SCENES))
def test_equals_oracle(name):
    grid, iso = ORACLE_SCENES[name]()
    verts, faces = mc(torch.from_numpy(grid).to(DEV), iso)
    check_against_oracle(grid, iso, verts, faces)


@pytest.mark.parametrize("n", [4, 5, 202])
def test_every_voxel_is_processed(n):
    """The reference drops the last voxels of these sizes, on the far side along dim 0; here the
    surface is whole and equals the corrected restatement."""
    grid = (sphere(n) < 1.2).astype(np.uint8)[None] if n > 5 else np.ones((1, n, n, n), np.uint8)
    verts, faces = mc(torch.from_numpy(grid).to(DEV))
    check_against_oracle(grid, 0.5, verts, faces)
    assert as_np(verts[0])[:, 0].max() == n + 0.5    # the far side along dim 0 is there


@pytest.mark.parametrize("name", list(QUIRKS))
def test_deviations_from_recorded_reference(name):
    """Where the reference's operator drops voxels, scrambles a non-cubic grid's strides or caps its
    vertices (recorded from it), the output here differs from it and equals the corrected restatement."""
    grid, iso, ref = reference(name, QUIRKS)
    verts, faces = mc(torch.from_numpy(grid).to(DEV), iso)
    check_against_oracle(grid, iso, verts, faces)
    assert not (ref.equal("v0", verts[0]) and ref.equal("f0", faces[0]))


def test_past_the_vertex_cap():
    """A checkerboard of side 40 has more vertices than the reference's cap of X*Y*100 - 3."""
    grid = checker(40)[None]
    verts, faces = mc(torch.from_numpy(grid).to(DEV))
    assert verts[0].shape[0] > 42 * 42 * 100 - 3
    check_against_oracle(grid, 0.5, verts, faces)
    assert int(faces[0].max()) == verts[0].shape[0] - 1 and int(faces[0].min()) == 0


def test_no_surface_and_empty_batch(capfd):
    for grid in (torch.zeros((2, 5, 6, 7), device=DEV), torch.full((1, 4, 4, 4), 0.2, device=DEV)):
        verts, faces = mc(grid)
        assert all(v.shape == (0, 3) and v.dtype == torch.float32 for v in verts)
        assert all(f.shape == (0, 3) and f.dtype == torch.int64 for f in faces)
    assert mc(torch.zeros((0, 3, 3, 3), device=DEV)) == ([], [])
    v, f = mc(torch.ones((1, 0, 3, 3), device=DEV))
    assert v[0].shape == (0, 3) and f[0].shape == (0, 3)
    torch.cuda.synchronize()
    out = capfd.readouterr()
    assert out.out == "" and out.err == ""


@pytest.mark.parametrize("dtype", [torch.bool, torch.uint8, torch.int8, torch.int32, torch.int64, torch.float16,
                                   torch.bfloat16, torch.float64])
def test_dtypes_equal_their_float(dtype):
    rng = np.random.default_rng(21)
    base = torch.from_numpy(rng.integers(0, 3, (2, 11, 9, 13))).to(DEV)
    grid = (base > 0) if dtype == torch.bool else base.to(dtype)
    verts, faces = mc(grid, 0.5)
    rv, rf = mc(grid.float(), 0.5)
    for b in range(2):
        assert torch.equal(verts[b], rv[b]) and torch.equal(faces[b], rf[b])


def test_non_contiguous_input():
    rng = np.random.default_rng(22)
    big = torch.from_numpy(rng.random((3, 20, 18, 24)).astype(np.float32)).to(DEV)
    for grid in (big[::2, 1:17, :, ::2], big.permute(0, 3, 1, 2), big.transpose(1, 3)[:, 2:]):
        for g in (grid, (grid > 0.5).to(torch.uint8).transpose(2, 3).contiguous().transpose(2, 3)):
            assert not g.is_contiguous()
            verts, faces = mc(g, 0.4)
            rv, rf = mc(g.contiguous(), 0.4)
            for b in range(g.shape[0]):
                assert torch.equal(verts[b], rv[b]) and torch.equal(faces[b], rf[b])


def test_reruns_are_byte_identical():
    grid = torch.from_numpy(np.stack([occupancy(48, 23), occupancy(48, 24)])).to(DEV)
    runs = []
    for _ in range(3):
        g = grid.clone().requires_grad_(True)
        verts, faces = mc(g)
        flat = torch.cat(verts)
        flat.backward(torch.cos(flat * 3.0))
        runs.append((as_np(flat).tobytes(), as_np(torch.cat(faces)).tobytes(), as_np(g.grad).tobytes()))
    assert runs[0] == runs[1] == runs[2]


def test_one_sync_per_call_and_none_in_backward():
    grid = torch.from_numpy(np.stack([occupancy(24, 25), occupancy(24, 26), occupancy(24, 27)])).to(DEV)
    grid.requires_grad_(True)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            verts, faces = mc(grid)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [w for w in caught if "called a synchronizing" in str(w.message)]
    assert len(syncs) == 1, [str(w.message) for w in caught]
    flat = torch.cat(verts)
    g = torch.randn_like(flat)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        flat.backward(g)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert grid.grad is not None and grid.grad.shape == grid.shape


@pytest.mark.parametrize("name", ["smooth", "noisy", "views"])
def test_gradients_against_float64_autograd(name):
    """Gradients of sum(w * vertices) against the float64 restatement's autograd.  Each vertex's
    gradient is (t - 1) / (f1 - f0) or -t / (f1 - f0) times its weight: with |f1 - f0| >= 1e-3 the
    float32 relative error stays below ~1e-5 of the gradient's scale; scenes keep every edge's
    difference above that."""
    rng = np.random.default_rng({"smooth": 31, "noisy": 32, "views": 33}[name])
    if name == "smooth":
        grid = occupancy(20, 34)[None]
    elif name == "noisy":
        grid = rng.random((1, 14, 17, 11)).astype(np.float32)
    else:
        grid = np.stack([occupancy(16, 35), rng.random((16, 16, 16)).astype(np.float32)])
    grid = np.round(grid * 500) / 500 + 0.0007   # values on a 2e-3 lattice, off the iso value
    grid = grid.astype(np.float32)
    g = torch.from_numpy(grid).to(DEV).requires_grad_(True)
    verts, faces = mc(g, 0.5)
    ws = [torch.from_numpy(rng.standard_normal(tuple(v.shape))).to(DEV).float() for v in verts]
    sum((v * w).sum() for v, w in zip(verts, ws)).backward()
    for b in range(grid.shape[0]):
        ov, of, top = oracle(grid[b], 0.5)
        g64 = torch.from_numpy(grid[b].astype(np.float64)).requires_grad_(True)
        v64 = O.vertices_f64(g64, 0.5, top)
        assert np.abs(v64.detach().numpy() - ov).max() < 1e-5
        (v64 * torch.from_numpy(as_np(ws[b])).double()).sum().backward()
        ref = g64.grad.numpy()
        ours = as_np(g.grad[b])
        scale = np.abs(ref).max()
        assert scale > 0
        assert np.abs(ours - ref).max() <= 1e-5 * scale, (np.abs(ours - ref).max(), scale)


def test_float64_input_backpropagates_through_float():
    rng = np.random.default_rng(36)
    g = torch.from_numpy(rng.random((1, 9, 9, 9))).to(DEV).requires_grad_(True)
    verts, _ = mc(g)
    verts[0].sum().backward()
    g32 = g.detach().float().requires_grad_(True)
    v32, _ = mc(g32)
    v32[0].sum().backward()
    assert g.grad.dtype == torch.float64 and torch.equal(g.grad.float(), g32.grad)


def test_256_cubed_two_views_in_bounded_memory():
    """Peak memory of a 256^3 call with two views, from the header's layout: 17 bytes per padded cube
    (cases, scans and counts) plus the outputs, with 32 MB for the allocator's rounding."""
    n, B = 256, 2
    grid = torch.from_numpy(np.stack([(sphere(n) < 0.8), (sphere(n, (0.3, 0.2, -0.4)) < 0.5)]).astype(np.uint8))
    grid = grid.to(DEV)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    verts, faces = mc(grid)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    cubes = B * (n + 2) ** 3
    out = sum(v.numel() * 4 + f.numel() * 8 for v, f in zip(verts, faces))
    bound = 17 * cubes + 4 * (cubes // 4096 + 2) + out + 32 * 1024 * 1024
    assert peak <= bound, (peak, bound)
    for b in range(B):
        v1, f1 = mc(grid[b:b + 1])
        assert torch.equal(verts[b], v1[0]) and torch.equal(faces[b], f1[0])
        assert int(faces[b].min()) == 0 and int(faces[b].max()) == verts[b].shape[0] - 1


def test_workspace_at_an_odd_address(monkeypatch):
    """Every workspace starting at byte 1 of a larger buffer: the outputs of an aligned one."""
    grid = torch.from_numpy(np.stack([occupancy(24, 23), occupancy(24, 24)])).to(DEV)

    def run():
        verts, faces = mc(grid)
        return [torch.cat(verts), torch.cat(faces)]

    want = run()
    scratch, odd = _lib.scratch, []
    monkeypatch.setattr(_lib, "scratch", lambda n, device: odd.append(n) or scratch(int(n) + 1, device)[1:])
    got = run()
    assert odd
    for a, b in zip(want, got):
        assert torch.equal(a, b)
