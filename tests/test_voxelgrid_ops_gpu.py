"""kaolin.ops.voxelgrid on the GPU: bit-equal to the reference's outputs in tests/golden/voxelgrid.npz for
every accepted dtype and for strided input; fill equal to scipy's binary_fill_holes on large random and
voxelized grids, and to the known answer of large built scenes; extract_surface bit-equal to
F.avg_pool3d on CUDA; odms round trips; the documented deviations, errors and limits; reruns, host
reads, workspace alignment and peak memory."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from scipy import ndimage

from kaolin_b200 import _lib, synthetic
from kaolin_b200.ops import voxelgrid as vg
from kaolin_b200.ops.conversions import trianglemeshes_to_voxelgrids
from oracle import voxelgrid as ov
from test_voxelgrid_ops_cpu import FILL, ODMS, PROJECT, SURFACE, project_args

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def variants(t, dtypes):
    """t in each dtype (values kept), contiguous and as a permuted view of the same values."""
    for dt in dtypes:
        c = t.to(dt)
        yield c
        yield c.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)     # strides (XYZ, Y, 1, XY)


FILL_DTYPES = (torch.bool, torch.uint8, torch.float32, torch.float64, torch.int64, torch.int32)


@pytest.mark.parametrize("name", sorted(FILL))
def test_fill_equals_reference_golden(name):
    sc = FILL[name]
    g = cuda(sc["grid"])
    expect = torch.from_numpy(sc["out"])
    out = vg.fill(g)
    assert out.dtype == torch.bool and torch.equal(out.cpu(), expect)
    binary = g != 0
    for v in variants(binary, FILL_DTYPES):
        assert torch.equal(vg.fill(v).cpu(), expect), v.dtype


@pytest.mark.parametrize("mode", ["wide", "thin"])
@pytest.mark.parametrize("name", sorted(SURFACE))
def test_extract_surface_equals_reference_golden(name, mode):
    sc = SURFACE[name]
    g = cuda(sc["grid"])
    dtypes = (torch.bool, torch.float32, torch.float64) if g.dtype == torch.bool else (g.dtype, torch.float64)
    for v in variants(g, dtypes):
        out = vg.extract_surface(v, mode)
        assert out.dtype == torch.bool and torch.equal(out.cpu(), torch.from_numpy(sc[mode])), v.dtype


@pytest.mark.parametrize("name", sorted(ODMS))
def test_extract_odms_equals_reference_golden(name):
    sc = ODMS[name]
    g = cuda(sc["grid"])
    expect = torch.from_numpy(sc["out"])
    for v in [g] + list(variants(g != 0, FILL_DTYPES)):
        out = vg.extract_odms(v)
        assert out.dtype == torch.int64 and torch.equal(out.cpu(), expect), v.dtype


@pytest.mark.parametrize("name", sorted(PROJECT))
def test_project_odms_equals_reference_golden(name):
    odms, grid, votes = project_args(PROJECT[name])
    expect = torch.from_numpy(PROJECT[name]["out"])
    o = cuda(odms)
    for oo in (o, o.transpose(2, 3).contiguous().transpose(2, 3)):
        if grid is None:
            out = vg.project_odms(oo, votes=votes)
        else:
            g = cuda(grid)
            out = vg.project_odms(oo, g, votes)
            assert torch.equal(vg.project_odms(oo, g.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1),
                                               votes).cpu(), expect)
        assert out.dtype == torch.bool and torch.equal(out.cpu(), expect)


def test_project_odms_every_vote_and_odm_dtype_against_oracle():
    rng = np.random.default_rng(3)
    D = 24
    odms = rng.integers(0, D + 1, (2, 6, D, D))
    frac = rng.integers(-4, 4 * D + 8, (2, 6, D, D)) / 4
    grids = [None, rng.random((2, D, D, D)) < 0.6, rng.integers(0, 5, (2, D, D, D)).astype(np.uint8),
             (rng.integers(-4, 9, (2, D, D, D)) / 4).astype(np.float32), rng.integers(-4, 9, (2, D, D, D)) / 4]
    for votes in range(8):
        for o in (odms.astype(np.int64), odms.astype(np.int32), frac.astype(np.float32), frac):
            for g in grids:
                out = vg.project_odms(cuda(o), None if g is None else cuda(g), votes)
                np.testing.assert_array_equal(out.cpu().numpy(), ov.project_odms(o, g, votes))


def scipy_fill(grid):
    return np.stack([ndimage.binary_fill_holes(v) for v in grid.cpu().numpy()])


def test_fill_equals_scipy_near_percolation():
    g = torch.rand((8, 128, 128, 128), device=DEV, generator=torch.Generator(DEV).manual_seed(5)) < 0.69
    np.testing.assert_array_equal(vg.fill(g).cpu().numpy(), scipy_fill(g))


def test_fill_equals_scipy_on_voxelized_icospheres():
    v, f = synthetic.icosphere(5)
    rng = np.random.default_rng(1)
    views = np.stack([v * rng.uniform(0.6, 1.0) + rng.normal(scale=0.1, size=3) for _ in range(4)])
    g = trianglemeshes_to_voxelgrids(cuda(views.astype(np.float32)), cuda(f), 256)
    out = vg.fill(g)
    np.testing.assert_array_equal(out.cpu().numpy(), scipy_fill(g != 0))
    assert out.sum() > 2 * (g != 0).sum()        # the shells were filled


def serpentine(n, dev=DEV):
    """A solid n^3 grid with one tunnel: on every other z plane it snakes along x through every other y
    row, turning at alternate ends; it climbs to the next plane at alternate ends of the snake and
    opens on the face x = 0.  The tunnel is the only empty space, so fill must keep all of it."""
    g = torch.ones((n, n, n), dtype=torch.bool, device=dev)
    rows = torch.arange(1, n - 1, 2, device=dev)
    planes = torch.arange(1, n - 1, 2, device=dev)
    turn_x = torch.where(torch.arange(len(rows) - 1, device=dev) % 2 == 0, n - 2, 1)
    end = (n - 2 if (len(rows) - 1) % 2 == 0 else 1, int(rows[-1]))
    for p, z in enumerate(planes.tolist()):
        g[1:n - 1, rows, z] = False
        g[turn_x, rows[:-1] + 1, z] = False
        if p + 1 < len(planes):
            x, y = end if p % 2 == 0 else (1, 1)
            g[x, y, z + 1] = False
    g[0, 1, 1] = False
    return g


def test_fill_serpentine_512_keeps_the_tunnel():
    g = serpentine(512)
    out = vg.fill(g[None])[0]
    assert torch.equal(out, g)                           # nothing filled: the tunnel reaches the border
    closed = g.clone()
    closed[0, 1, 1] = True                               # seal the mouth: the whole tunnel is filled
    assert bool(vg.fill(closed[None]).all())


def test_fill_nested_boxes_1024_and_peak_memory():
    """Hollow one-voxel boxes nested 48 voxels apart in one 1024^3 view; the second is opened by a
    one-voxel tunnel.  While the outer box is closed everything inside it fills; once it is opened too,
    the two gaps the tunnels join stay empty and the third box's inside fills."""
    n = 1024
    g = torch.zeros((1, n, n, n), dtype=torch.bool, device=DEV)
    for lo in range(8, 400, 48):
        g[0, lo:n - lo, lo:n - lo, lo:n - lo] = True
        g[0, lo + 1:n - lo - 1, lo + 1:n - lo - 1, lo + 1:n - lo - 1] = False
    g[0, 56, 500, 500] = False
    torch.cuda.synchronize()
    ws = _lib.voxelgrid_fill_workspace_bytes(1, n, n, n, "fill")
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = vg.fill(g)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak <= n ** 3 + ws + (1 << 21), (peak, ws)
    assert bool(out[0, 8:n - 8, 8:n - 8, 8:n - 8].all())
    assert not bool(out[0, :8].any()) and not bool(out[0, n - 8:].any())
    del out
    g[0, 8, 500, 500] = False
    out = vg.fill(g)
    assert not bool(out[0, 9:104, 500, 500].any())
    assert bool(out[0, 104:n - 104, 104:n - 104, 104:n - 104].all())


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_extract_surface_bit_equal_to_avg_pool3d(dtype):
    gen = torch.Generator(DEV).manual_seed(7)
    g = torch.rand((2, 128, 128, 128), device=DEV, dtype=dtype, generator=gen) * 1.5
    g[torch.rand(g.shape, device=DEV, generator=gen) < 0.3] = 0
    g[torch.rand(g.shape, device=DEV, generator=gen) < 0.3] = 1
    x = g.unsqueeze(1)
    wide = (F.avg_pool3d(x, 3, padding=1, stride=1).squeeze(1) < 1) * g.bool()
    thin = ((F.avg_pool3d(x, (3, 1, 1), padding=(1, 0, 0), stride=1).squeeze(1) < 1)
            | (F.avg_pool3d(x, (1, 3, 1), padding=(0, 1, 0), stride=1).squeeze(1) < 1)
            | (F.avg_pool3d(x, (1, 1, 3), padding=(0, 0, 1), stride=1).squeeze(1) < 1)) * g.bool()
    assert torch.equal(vg.extract_surface(g, "wide"), wide)
    assert torch.equal(vg.extract_surface(g, "thin"), thin)


def test_odms_round_trip_on_voxelized_meshes():
    v, f = synthetic.icosphere(4)
    rng = np.random.default_rng(2)
    views = np.stack([v * rng.uniform(0.5, 1.0) + rng.normal(scale=0.1, size=3) for _ in range(3)])
    g = vg.fill(trianglemeshes_to_voxelgrids(cuda(views.astype(np.float32)), cuda(f), 64))
    odms = vg.extract_odms(g)
    np.testing.assert_array_equal(odms.cpu().numpy(), ov.extract_odms(g.cpu().numpy()))
    carved = vg.project_odms(odms)
    assert bool((carved | ~g).all())                     # the visual hull holds the solid
    assert torch.equal(vg.extract_odms(carved), odms)    # and has the same depth maps
    assert torch.equal(vg.project_odms(odms, g), g)


def test_deviations_and_errors():
    assert vg.fill(torch.zeros((0, 4, 4, 4), device=DEV)).shape == (0, 4, 4, 4)
    assert vg.fill(torch.zeros((2, 4, 0, 4), device=DEV)).shape == (2, 4, 0, 4)
    assert vg.extract_surface(torch.zeros((0, 3, 3, 3), device=DEV)).shape == (0, 3, 3, 3)
    assert vg.extract_odms(torch.zeros((0, 3, 3, 3), device=DEV)).shape == (0, 6, 3, 3)
    assert vg.project_odms(torch.zeros((0, 6, 3, 3), device=DEV)).shape == (0, 3, 3, 3)
    g = torch.ones((1, 3, 3, 3), device=DEV)
    for f in (vg.fill, vg.extract_surface, vg.extract_odms):
        with pytest.raises(ValueError):
            f(g[0])
    with pytest.raises(ValueError):
        vg.extract_surface(g, "narrow")
    for dt in (torch.float16, torch.bfloat16, torch.uint8, torch.int64):
        with pytest.raises(TypeError):
            vg.extract_surface(g.to(dt))
    with pytest.raises(ValueError):
        vg.extract_odms(torch.ones((1, 3, 3, 4), device=DEV))
    odms = torch.zeros((1, 6, 3, 3), dtype=torch.int64, device=DEV)
    with pytest.raises(ValueError):
        vg.project_odms(odms[:, :5])
    with pytest.raises(ValueError):
        vg.project_odms(odms, torch.ones((2, 3, 3, 3), dtype=torch.bool, device=DEV))
    with pytest.raises(ValueError):
        vg.project_odms(odms, torch.ones((1, 3, 3, 4), dtype=torch.bool, device=DEV))
    with pytest.raises(TypeError):
        vg.project_odms(odms.to(torch.int16))
    with pytest.raises(TypeError):
        vg.project_odms(odms, torch.ones((1, 3, 3, 3), dtype=torch.int64, device=DEV))
    assert torch.equal(vg.downsample(torch.ones((1, 4, 4, 4), dtype=torch.bool, device=DEV), 2),
                       torch.ones((1, 2, 2, 2), dtype=torch.half, device=DEV))
    with pytest.raises(ValueError):
        vg.downsample(torch.ones((1, 4, 4, 4), device=DEV), [2, 2])


def test_per_view_size_limit():
    big = torch.ones((1, 1, 1, 1), dtype=torch.bool, device=DEV).expand(1, 1291, 1291, 1291)
    with pytest.raises(RuntimeError, match="fill"):
        vg.fill(big)
    with pytest.raises(RuntimeError, match="extract_surface"):
        vg.extract_surface(big)
    with pytest.raises(RuntimeError, match="extract_odms"):
        vg.extract_odms(big)


def test_reruns_are_byte_identical_and_make_no_host_read():
    g = torch.rand((4, 96, 96, 96), device=DEV, generator=torch.Generator(DEV).manual_seed(9)) < 0.69
    odms = vg.extract_odms(g)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = [vg.fill(g), vg.extract_surface(g), vg.extract_surface(g, "thin"), vg.extract_odms(g),
             vg.project_odms(odms), vg.project_odms(odms, g, 2), vg.downsample(g, 2)]
        b = [vg.fill(g), vg.extract_surface(g), vg.extract_surface(g, "thin"), vg.extract_odms(g),
             vg.project_odms(odms), vg.project_odms(odms, g, 2), vg.downsample(g, 2)]
    finally:
        torch.cuda.set_sync_debug_mode("default")
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("offset", [1, 3, 255])
def test_workspace_at_an_odd_address(offset):
    g = (torch.rand((2, 40, 33, 57), device=DEV, generator=torch.Generator(DEV).manual_seed(4)) < 0.69)
    B, X, Y, Z = g.shape
    nbytes = _lib.voxelgrid_fill_workspace_bytes(B, X, Y, Z, "fill")
    ws = torch.empty(nbytes + offset, dtype=torch.uint8, device=DEV)[offset:]
    out = torch.empty_like(g)
    _lib.call("dibr_b200_voxelgrid_fill", DEV, B, X, Y, Z, _lib.DTYPE_U8, g.view(torch.uint8), *g.stride(), out, ws,
              nbytes, what="fill")
    np.testing.assert_array_equal(out.cpu().numpy(), scipy_fill(g))
    with pytest.raises(RuntimeError, match="workspace"):
        _lib.call("dibr_b200_voxelgrid_fill", DEV, B, X, Y, Z, _lib.DTYPE_U8, g.view(torch.uint8), *g.stride(), out,
                  ws, nbytes - 1, what="fill")
