"""DefTet sparse render (kaolin_b200/csrc/deftet.cu) against the reference's own CUDA operator
(``deftet_sparse_render_{forward,backward}_cuda``, oracle/build_ref_deftet.py), through its stored
outputs (tests/golden/ref_cuda_deftet.npz, oracle/ref_golden_deftet.py).

The forward must be bit-identical: face_idx, pixel_depth, w0 and w1 including the padding.  The
scenes are constructed, not sampled, around the places the binning of deftet.cu switches path or could
drop a hit: points and face bounding boxes exactly on cell borders of the view's G x G grid, shared
edges and vertices, depth-range limits, G = 8 .. 256 (the scan carried over up to 64 passes), faces of
16 and 17-20 cells (the wide list), 127/128/129/400 hits (the in-buffer sort and the ordered
fallback) and degenerate input.  Each case asserts, with a host restatement of the binning, that it
reaches what it was built for.  The backward gets the same face_idx and the weights
``deftet_sparse_render`` builds; it must be bit-identical where no two atomics meet, and within 1e-6
of the gradient's scale elsewhere (atomics order)."""
import numpy as np
import pytest
import torch

from oracle import build_ref_deftet, ref_golden_deftet
from kaolin_b200 import _C as b200_C

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 1e-8
FWD = ("fidx", "depth", "w0", "w1")
BWD = ("g_fvi", "g_ff")
SAME = 1e-6              # atomics-order allowance, of the gradient's scale
FULL_ROWS = 4096         # forward outputs of at most this many points are stored whole; larger
                         # outputs and the gradients keep digest, scale and a row sample (ref_golden)

f32 = np.float32


# ---- host restatement of deftet.cu's binning (float32 throughout, as the kernels compute it) ----

def grid_side(F):
    G = 8
    while G < 256 and G * G < F:
        G += 8
    return G


def view_bounds(pix, G):
    """deftet_bounds_kernel for one view: xmin, ymin, G / width, G / height (fminf/fmaxf skip NaN)."""
    x, y = pix[:, 0].astype(f32), pix[:, 1].astype(f32)
    x0, x1 = np.fmin.reduce(x, initial=np.inf), np.fmax.reduce(x, initial=-np.inf)
    y0, y1 = np.fmin.reduce(y, initial=np.inf), np.fmax.reduce(y, initial=-np.inf)
    if not (x1 >= x0) or not (y1 >= y0):
        x0 = y0 = f32(0); x1 = y1 = f32(1)
    wx, wy = np.fmax(f32(x1 - x0), f32(1e-20)), np.fmax(f32(y1 - y0), f32(1e-20))
    return f32(x0), f32(y0), f32(f32(G) / wx), f32(f32(G) / wy)


def cell_coord(v, lo, inv):
    with np.errstate(invalid="ignore", over="ignore"):
        return f32(np.asarray(v, f32) - lo) * inv


def cell_of(v, lo, inv, G):
    with np.errstate(invalid="ignore"):
        return np.fmin(np.fmax(cell_coord(v, lo, inv), f32(0)), f32(G - 1)).astype(np.int64)


def binning(s):
    """Per view: G, the points' cells, how many points sit exactly on an inner cell border, and each
    face's cell count (0 for an empty or NaN box) — deftet_bin_kernel's decisions."""
    B, F = s["fvz"].shape[:2]
    G = grid_side(F)
    out = []
    for b in range(B):
        lo_x, lo_y, ix, iy = view_bounds(s["pix"][b], G)
        px, py = s["pix"][b, :, 0], s["pix"][b, :, 1]
        cx, cy = cell_coord(px, lo_x, ix), cell_coord(py, lo_y, iy)
        on_border = lambda c: np.isfinite(c) & (c == np.floor(c)) & (c >= 1) & (c <= G - 1)
        cell = cell_of(py, lo_y, iy, G) * G + cell_of(px, lo_x, ix, G)
        bb = s["bb"][b]
        with np.errstate(invalid="ignore"):
            ok = (bb[:, 2] > bb[:, 0]) & (bb[:, 3] > bb[:, 1])
        nx = cell_of(bb[:, 2], lo_x, ix, G) - cell_of(bb[:, 0], lo_x, ix, G) + 1
        ny = cell_of(bb[:, 3], lo_y, iy, G) - cell_of(bb[:, 1], lo_y, iy, G) + 1
        out.append(dict(G=G, cell=cell, border=int((on_border(cx) | on_border(cy)).sum()),
                        ncells=np.where(ok, nx * ny, 0), bounds=(lo_x, lo_y, ix, iy)))
    return out


# ---- scenes ----

def _scene(fvi, fvz, pix, rr):
    fvi = np.ascontiguousarray(fvi, f32)
    with np.errstate(invalid="ignore"):
        bb = np.concatenate([fvi.min(2), fvi.max(2)], -1)          # what deftet_sparse_render passes
    return dict(fvz=np.ascontiguousarray(fvz, f32), fvi=fvi, bb=np.ascontiguousarray(bb, f32),
                pix=np.ascontiguousarray(pix, f32), rr=np.ascontiguousarray(rr, f32))


def _wide_range(B, P):
    return np.broadcast_to(np.array([-10.0, 10.0], f32), (B, P, 2))


def lattice_scene():
    """16 x 16 squares of side 3, two triangles each, on integer points 0..48 (= 2G + 1 per axis,
    G = 24): every even coordinate is a cell border, every mesh vertex is a point, bounding boxes start
    and end on points, points lie on shared edges and vertices.  View 1 has the other winding."""
    n, side = 16, 3
    v = np.stack(np.meshgrid(np.arange(n + 1) * side, np.arange(n + 1) * side, indexing="xy"), -1).astype(f32)
    z = -(1.0 + 0.01 * v[..., 0] + 0.02 * v[..., 1]).astype(f32)
    tri, tz = [], []
    for j in range(n):
        for i in range(n):
            a, b, c, d = (j, i), (j, i + 1), (j + 1, i + 1), (j + 1, i)
            for t in ((a, b, c), (a, c, d)):
                tri.append([v[k] for k in t]); tz.append([z[k] for k in t])
    tri, tz = np.array(tri, f32), np.array(tz, f32)
    fvi = np.stack([tri, tri[:, [0, 2, 1]]])
    fvz = np.stack([tz, tz[:, [0, 2, 1]]])
    g = np.arange(n * side + 1, dtype=f32)
    pts = np.stack(np.meshgrid(g, g, indexing="xy"), -1).reshape(-1, 2)
    pix = np.stack([pts, pts])
    return _scene(fvi, fvz, pix, _wide_range(2, pts.shape[0]))


DEPTH_LAYERS = np.array([0.0, -1.0, -1.5, -2.7, 0.3, -0.1], f32)


def depth_scene():
    """Six layers of the same two triangles at constant z; per point a range whose dmin or dmax is a
    layer's z, an empty range (dmin == dmax), an inverted one, or the one-ulp window around z."""
    L = len(DEPTH_LAYERS)
    sq = np.array([[[0, 0], [4, 0], [4, 4]], [[0, 0], [4, 4], [0, 4]]], f32)
    fvi = np.concatenate([sq] * L)[None]
    fvz = np.repeat(DEPTH_LAYERS, 2)[:, None].repeat(3, 1)[None]
    rng = np.random.default_rng(11)
    P = 203
    pix = rng.uniform(0.05, 3.95, (1, P, 2)).astype(f32)
    rr = np.zeros((1, P, 2), f32)
    for p in range(P):
        zl = DEPTH_LAYERS[(p // 5) % L]
        rr[0, p] = [(zl, zl + 0.05), (zl - 0.05, zl), (zl, zl), (zl + 0.25, zl - 0.25),
                    (np.nextafter(zl, f32(-np.inf)), np.nextafter(zl, f32(np.inf)))][p % 5]
    return _scene(fvi, fvz, pix, rr)


def grid_scene(F):
    """F small faces (1.5 cells across, half with integer vertices) over integer points 0..2G: half of
    the point coordinates are cell borders; points cover every cell row of the grid."""
    G = grid_side(F)
    rng = np.random.default_rng(F)
    span = 2 * G
    c = rng.uniform(0, span, (F, 1, 2))
    fvi = c + rng.uniform(-1.5, 1.5, (F, 3, 2))
    fvi[: F // 2] = np.round(fvi[: F // 2])
    fvz = -rng.uniform(1, 3, (F, 3))
    P = 3003
    pts = rng.integers(0, span + 1, (P, 2)).astype(f32)
    pts[:2] = [[0, 0], [span, span]]
    pts[2:2 + span + 1, 1] = np.arange(span + 1)                    # one point in every row of cells
    pts[P // 2:] += rng.uniform(0, 1, (P - P // 2, 2)).astype(f32) * (rng.uniform(size=(P - P // 2, 1)) < 0.5)
    pts = np.clip(pts, 0, span)
    return _scene(fvi[None], fvz[None], pts[None], _wide_range(1, P))


WIDE_SHAPES = [(4, 4), (2, 8), (8, 2), (1, 16), (16, 1), (1, 17), (17, 1), (3, 6), (6, 3), (4, 5), (5, 4)]


def wide_scene():
    """G = 32 over points 0..64 (cells 2 wide): right triangles whose bounding boxes cover exactly
    a x b cells for the shapes above, some ending exactly on a cell border (one more cell), in both
    orientations, among small faces inside one cell."""
    F = 1000
    rng = np.random.default_rng(7)
    tris = []
    for k in range(20):
        for (a, b) in WIDE_SHAPES:
            cx, cy = rng.integers(0, 32 - a + 1), rng.integers(0, 32 - b + 1)
            x0, y0 = 2 * cx + 0.5, 2 * cy + 0.5
            x1, y1 = 2 * (cx + a - 1) + 1.5, 2 * (cy + b - 1) + 1.5
            if k % 4 == 3:
                x0, y0 = 2.0 * cx, 2.0 * cy                             # starts on a border
            if k % 4 == 2 and cx + a < 32:
                x1 = 2.0 * (cx + a)                                      # ends on a border: + 1 column
            tris.append([[x0, y0], [x1, y0], [x0, y1]] if k % 2 else [[x1, y1], [x0, y1], [x1, y0]])
    n_big = len(tris)
    c = rng.integers(0, 32, (F - n_big, 1, 2)) * 2 + 0.2
    small = c + rng.uniform(0, 1.6, (F - n_big, 3, 2))
    fvi = np.concatenate([np.array(tris, f32), small.astype(f32)])
    perm = rng.permutation(F)
    fvi = fvi[perm]
    fvz = -rng.uniform(1, 3, (F, 3))
    g = np.arange(65, dtype=f32)
    pts = np.stack(np.meshgrid(g, g, indexing="xy"), -1).reshape(-1, 2)
    pts = np.concatenate([pts, rng.uniform(0, 64, (777, 2)).astype(f32)])
    return _scene(fvi[None], fvz[None], pts[None], _wide_range(1, pts.shape[0])), perm < n_big


HIT_GROUPS = [0, 1, 31, 32, 33, 127, 128, 129, 400]


def hits_scene():
    """A stack of h slightly different triangles around each of nine centres, h in HIT_GROUPS, the
    faces of all stacks interleaved in index order; four points near each centre lie in all h, two
    more in none.  Most faces go to the cell lists."""
    rng = np.random.default_rng(3)
    base = np.array([[0.0, 0.9], [-0.8, -0.5], [0.8, -0.5]])
    tris, group = [], []
    for gi, h in enumerate(HIT_GROUPS):
        ctr = np.array([10.0 * gi, 5.0])
        for k in range(h):
            tris.append(ctr + base * (1 + 0.3 * rng.uniform()) + rng.uniform(-0.05, 0.05, 2))
            group.append(gi)
    tris = np.array(tris, f32)
    perm = rng.permutation(len(tris))
    fvi = tris[perm]
    fvz = -rng.uniform(1, 3, (len(tris), 3))
    pts = []
    for gi, _ in enumerate(HIT_GROUPS):
        for k in range(4):
            pts.append([10.0 * gi + rng.uniform(-0.03, 0.03), 5.0 + rng.uniform(-0.03, 0.03)])
    pts.extend([[-5.0, 0.0], [85.0, 10.0]])                            # give the grid a 2-D extent
    pts = np.array(pts, f32)
    return _scene(fvi[None], fvz[None], pts[None], _wide_range(1, len(pts)))


def degenerate_scene():
    """Five views of 64 faces and 100 points each:
    0 collinear, zero-area, single-point, NaN and +-inf faces (and a NaN depth) among normal ones,
      points on the collinear faces' lines;
    1 points with NaN and +-inf coordinates among normal points;
    2 all points identical (grid width clamped to 1e-20);
    3 points outside every face and faces outside every point (clamped to the border cells);
    4 point extents near 1e30, small faces near the origin and faces 1e30 across."""
    rng = np.random.default_rng(5)
    F, P = 64, 100
    normal = lambda n, lo, hi: (rng.uniform(lo, hi, (n, 1, 2)) + rng.uniform(-0.3, 0.3, (n, 3, 2))).astype(f32)
    fvi = np.stack([normal(F, -1, 1) for _ in range(5)])
    fvz = -rng.uniform(1, 3, (5, F, 3)).astype(f32)
    pix = rng.uniform(-1, 1, (5, P, 2)).astype(f32)
    # view 0
    t = rng.uniform(-1, 1, (8, 1, 1)).astype(f32)
    fvi[0, 0:8] = t + np.array([[0, 0], [0.5, 0.5], [1, 1]], f32)          # collinear, on a diagonal
    fvi[0, 8:12, 1] = fvi[0, 8:12, 0]                                       # two equal vertices
    fvi[0, 12:16] = fvi[0, 12:16, :1]                                       # all three equal
    fvi[0, 16, 0, 0] = np.nan; fvi[0, 17, 1, 1] = np.nan
    fvi[0, 18, 2, 0] = np.inf; fvi[0, 19, 0, 1] = -np.inf; fvi[0, 20, 1, 0] = -np.inf; fvi[0, 21, 2, 1] = np.inf
    fvz[0, 22, 1] = np.nan
    pix[0, :16] = (t[:, 0] + np.array([[0.25, 0.25], [0.5, 0.5]], f32)[:, None]).reshape(16, 2)
    # view 1
    pix[1, 0:10, 0] = np.nan; pix[1, 10:15, 1] = np.nan
    pix[1, 15:20, 0] = np.inf; pix[1, 20:25, 1] = -np.inf
    # view 2
    pix[2] = [0.1, -0.2]
    # view 3
    pix[3] = rng.uniform(-0.5, 0.5, (P, 2))
    fvi[3, :32] += np.array([3.0, 0.0], f32); fvi[3, 32:48] -= np.array([0.0, 3.0], f32)
    fvi[3, 48:] += np.array([-3.0, 3.0], f32)
    # view 4
    pix[4, 0] = [-1e30, -1e30]; pix[4, 1] = [1e30, 1e30]; pix[4, 2:10] = rng.uniform(-1e30, 1e30, (8, 2))
    fvi[4, :8] = rng.uniform(-1e30, 1e30, (8, 3, 2))
    rr = np.broadcast_to(np.array([-10.0, 10.0], f32), (5, P, 2)).copy()
    return _scene(fvi, fvz, pix, rr)


def shapes_scene(B, F, P, seed):
    """B views with point extents 1, 100 and 0.01 and small faces of the same spread."""
    rng = np.random.default_rng(seed)
    scale = np.array([1.0, 100.0, 0.01, 7.0])[:B, None, None, None]
    fvi = ((rng.uniform(-1, 1, (B, F, 1, 2)) + rng.uniform(-0.2, 0.2, (B, F, 3, 2))) * scale).astype(f32)
    fvz = -rng.uniform(1, 3, (B, F, 3))
    pix = (rng.uniform(-1, 1, (B, P, 2)) * scale[:, :, 0]).astype(f32)
    return _scene(fvi, fvz, pix, _wide_range(B, P))


def exact_scene():
    """One small triangle per lattice cell with one point strictly inside it: every face is hit by
    at most one (point, k) entry, so no two atomics of the backward meet."""
    rng = np.random.default_rng(13)
    n = 24
    ij = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="xy"), -1).reshape(-1, 1, 2)
    base = np.array([[0.1, 0.1], [0.9, 0.15], [0.3, 0.85]])
    fvi = (ij + base + rng.uniform(-0.05, 0.05, (n * n, 3, 2))).astype(f32)
    fvz = -rng.uniform(1, 3, (n * n, 3))
    pts = (ij[:, 0] + np.array([0.42, 0.36]) + rng.uniform(-0.04, 0.04, (n * n, 2))).astype(f32)
    pts = pts[: n * n - 37]                                                 # some faces without a point
    return _scene(fvi[None], fvz[None], pts[None], _wide_range(1, len(pts)))


# ---- running both operators ----

def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int32) if a.dtype == np.float32 else a


def forward(case, s, knum):
    args = [T(s[k]) for k in ("fvz", "fvi", "bb", "pix", "rr")]

    def live():
        C = build_ref_deftet.load()
        assert C is not None, "oracle/_ref/kaolin_ref_deftet_C.so is needed to record"
        return dict(zip(FWD, C.deftet_sparse_render_forward_cuda(*args, knum, EPS)))

    B, P = s["pix"].shape[:2]
    ref = ref_golden_deftet.reference(case, live, FWD, full=FWD if B * P <= FULL_ROWS else ())
    ours = b200_C.render.mesh.deftet_sparse_render_forward_cuda(*args, knum, EPS)
    torch.cuda.synchronize()
    return ref, dict(zip(FWD, ours))


def assert_forward_identical(case, ref, ours):
    for name in FWD:
        if ref.equal(name, ours[name]):
            continue
        mine, theirs = ref.pair(name, ours[name])
        bad = np.flatnonzero((_bits(mine) != _bits(theirs)).any(1))
        rows = ref.rows(name)[bad[:3]] if bad.size else []
        raise AssertionError(f"{case}: {name} differs from the reference operator"
                             + (f" at points {list(rows)} (of {bad.size} stored rows): ours "
                                f"{mine[bad[0]].tolist()} reference {theirs[bad[0]].tolist()}" if bad.size else
                                " outside the stored rows"))


def run_forward(case, s, knum):
    ref, ours = forward(case, s, knum)
    assert_forward_identical(case, ref, ours)
    out = {k: v.cpu().numpy() for k, v in ours.items()}
    out["hits"] = (out["fidx"] >= 0).sum(-1)
    return out


# ---- forward cases ----

def test_lattice_borders_shared_edges_and_both_windings():
    s = lattice_scene()
    o = run_forward("lattice", s, 8)
    info = binning(s)
    fidx, w0, w1 = o["fidx"], o["w0"], o["w1"]
    on_edge = (fidx >= 0) & ((w0 == 0) | (w1 == 0) | (w0 + w1 >= 1))
    print(f"\n[lattice] G {info[0]['G']}, points on a cell border {info[0]['border']}/{s['pix'].shape[1]}, "
          f"hits per point {np.bincount(o['hits'].ravel()).tolist()}, hits with a zero weight {int(on_edge.sum())}")
    assert info[0]["G"] == 24 and info[0]["border"] > s["pix"].shape[1] // 2
    assert (o["hits"] == 2).sum() > 0 and (o["hits"] == 1).sum() > 0 and on_edge.sum() > 0
    # bounding boxes start and end on points: the half-open test keeps a vertex only in the faces
    # whose box starts there
    assert (o["hits"][:, -1] == 0).all() and (o["hits"][0] == o["hits"][1]).all()


def test_depth_range_limits():
    s = depth_scene()
    o = run_forward("depth_limits", s, 16)
    L = len(DEPTH_LAYERS)
    kind = np.arange(s["pix"].shape[1]) % 5
    layer = DEPTH_LAYERS[(np.arange(s["pix"].shape[1]) // 5) % L]
    fidx, d = o["fidx"][0], o["depth"][0]
    layer_of = lambda f: DEPTH_LAYERS[f // 2]
    zero = layer == 0
    in_zero_layer = np.array([(layer_of(f[f >= 0]) == 0).any() for f in fidx])
    exact = np.isin(d, DEPTH_LAYERS).sum()
    print(f"\n[depth_limits] hits {int(o['hits'].sum())}, depths exactly a layer's z {exact}/{int(o['hits'].sum())}")
    assert (o["hits"][0][(kind == 2) | (kind == 3)] == 0).all()             # empty and inverted ranges
    assert in_zero_layer[zero & (kind == 0)].all()                         # dmin == z is included
    assert not in_zero_layer[zero & (kind == 1)].any()                     # dmax == z is excluded
    assert in_zero_layer[zero & (kind == 4)].all()


@pytest.mark.parametrize("F,G", [(64, 8), (65, 16), (4096, 64), (4097, 72), (65536, 256), (70000, 256)])
def test_grid_sizes(F, G):
    s = grid_scene(F)
    o = run_forward(f"grid_F{F}", s, 4)
    info = binning(s)[0]
    passes = -(-G * G // 1024)
    late = int(((info["cell"] >= 1024) & (o["hits"][0] > 0)).sum())
    print(f"\n[grid F={F}] G {info['G']}, scan passes {passes}, points on a cell border {info['border']}, "
          f"wide list {int((info['ncells'] > 16).sum())}, hit points in cells >= 1024: {late}, "
          f"hits per point mean {o['hits'].mean():.2f} max {o['hits'].max()}")
    assert info["G"] == G and info["border"] > 1000 and (o["hits"] > 0).sum() > 100
    if passes > 1:
        assert late > 100


def test_wide_list_boundary():
    s, big = wide_scene()
    o = run_forward("wide_list", s, 32)
    info = binning(s)[0]
    nc = info["ncells"]
    fidx = o["fidx"][0]
    hit16 = np.array([(nc[f[f >= 0]] == 16).any() for f in fidx])
    hit17 = np.array([((nc[f[f >= 0]] >= 17) & (nc[f[f >= 0]] <= 20)).any() for f in fidx])
    print(f"\n[wide_list] G {info['G']}, faces of 16 cells {int((nc == 16).sum())}, of 17-20 cells "
          f"{int(((nc >= 17) & (nc <= 20)).sum())}, wide list {int((nc > 16).sum())}, points hit by both "
          f"{int((hit16 & hit17).sum())}, hits per point max {o['hits'].max()}")
    assert info["G"] == 32 and (nc == 16).sum() >= 40 and ((nc >= 17) & (nc <= 20)).sum() >= 40
    assert (nc[~big] <= 4).all() and (o["hits"] < 32).all()
    assert (hit16 & hit17).sum() > 0


@pytest.mark.parametrize("knum", [1, 31, 32, 33, 128, 300])
def test_hit_count_boundary(knum):
    s = hits_scene()
    o = run_forward(f"hits_k{knum}", s, knum)
    want = np.concatenate([np.repeat(HIT_GROUPS, 4), [0, 0]])
    nc = binning(s)[0]["ncells"]
    print(f"\n[hits knum={knum}] hits per point {o['hits'][0][::4].tolist()}, ordered fallback for "
          f"{int((want > 128).sum())} points, wide list {int((nc > 16).sum())} of {nc.size}")
    assert (nc > 16).mean() < 0.5
    assert (o["hits"][0] == np.minimum(want, knum)).all()
    fidx = o["fidx"][0]
    assert all((np.diff(f[f >= 0]) > 0).all() for f in fidx)                 # index order


def test_degenerate_input():
    s = degenerate_scene()
    o = run_forward("degenerate", s, 8)
    info = binning(s)
    h, fidx, w0, w1 = o["hits"], o["fidx"], o["w0"], o["w1"]
    collinear = (fidx[0, :16] >= 0) & (fidx[0, :16] < 8) & (w0[0, :16] == 0) & (w1[0, :16] == 0)
    print(f"\n[degenerate] hits per view {h.sum(1).tolist()}, all-zero-weight hits on collinear faces "
          f"{int(collinear.sum())}, cells per unit in x {[float(info[b]['bounds'][2]) for b in range(5)]}")
    assert collinear.any()
    assert not np.isin(fidx[0], np.arange(12, 23)).any()                    # empty box, NaN, inf, NaN depth
    assert (h[1, :25] == 0).all() and (h[1, 25:] > 0).any()
    assert info[2]["bounds"][2] == f32(info[2]["G"]) / f32(1e-20)
    assert h[3].sum() == 0 and set(np.unique(info[3]["ncells"])) != {0}
    assert (h[4, :10] == 0).all() and h[4].sum() > 0


@pytest.mark.parametrize("B,F,P", [(3, 300, 37), (2, 100, 1), (2, 0, 45)])
def test_shapes(B, F, P):
    s = shapes_scene(B, F, P, seed=B * 1000 + F + P)
    o = run_forward(f"shapes_B{B}_F{F}_P{P}", s, 5)
    print(f"\n[shapes B={B} F={F} P={P}] hits per view {o['hits'].sum(1).tolist()}")
    assert o["fidx"].shape == (B, P, 5)
    if F == 0:
        assert (o["fidx"] == -1).all() and np.isneginf(o["depth"]).all()
    elif P > 1:
        assert (o["hits"].sum(1) > 0).all()


# ---- backward ----

def _scene_by_name(name):
    if name == "lattice":
        return lattice_scene(), 8
    if name.startswith("grid_F"):
        return grid_scene(int(name[6:])), 4
    if name.startswith("hits_k"):
        return hits_scene(), int(name[6:])
    if name == "degenerate":
        return degenerate_scene(), 8
    if name == "exact":
        return exact_scene(), 2
    raise KeyError(name)


def backward(case, s, knum, D, seed):
    ref_f, ours_f = forward(case, s, knum)
    assert ref_f.equal("fidx", ours_f["fidx"]), f"{case}: face_idx differs from the reference operator"
    idx, w0, w1 = ours_f["fidx"], ours_f["w0"], ours_f["w1"]
    w2 = (idx != -1).to(w0.dtype) - (w0 + w1)                         # as deftet_sparse_render builds it
    weights = torch.stack([w0, w1, w2], -1).contiguous()
    B, P, K = idx.shape
    F = s["fvi"].shape[1]
    rng = np.random.default_rng(seed)
    grad = T(rng.uniform(-1, 1, (B, P, K, D)).astype(f32))
    ff = T(rng.uniform(0, 1, (B, F, 3, D)).astype(f32))
    fvi = T(s["fvi"])

    def live():
        C = build_ref_deftet.load()
        assert C is not None, "oracle/_ref/kaolin_ref_deftet_C.so is needed to record"
        return dict(zip(BWD, C.deftet_sparse_render_backward_cuda(grad, idx, weights, fvi, ff, EPS)))

    ref = ref_golden_deftet.reference(f"{case}_bwd_D{D}", live, BWD)
    ours = b200_C.render.mesh.deftet_sparse_render_backward_cuda(grad, idx, weights, fvi, ff, EPS)
    return ref, dict(zip(BWD, ours)), idx.cpu().numpy()


def test_backward_bit_identical_where_no_atomics_meet():
    s, knum = _scene_by_name("exact")
    ref, ours, idx = backward("exact", s, knum, 1, seed=1)
    per_face = np.bincount(idx[idx >= 0], minlength=s["fvi"].shape[1])
    print(f"\n[exact] faces hit {int((per_face > 0).sum())}/{per_face.size}, most entries per face {per_face.max()}")
    assert per_face.max() == 1 and (per_face == 0).any()
    for name in BWD:
        assert ref.equal(name, ours[name]), f"{name} differs from the reference operator"


@pytest.mark.parametrize("D", [1, 3, 8])
@pytest.mark.parametrize("case", ["lattice", "grid_F4097", "grid_F70000", "hits_k128", "hits_k300", "degenerate"])
def test_backward_within_atomics_order(case, D):
    s, knum = _scene_by_name(case)
    ref, ours, idx = backward(case, s, knum, D, seed=D)
    F = s["fvi"].shape[1]
    for name in BWD:
        mine, theirs = ref.pair(name, ours[name])
        mine, theirs = mine.astype(np.float64), theirs.astype(np.float64)
        assert (np.isnan(mine) == np.isnan(theirs)).all(), (case, name, "NaN pattern")
        fin = np.isfinite(theirs)
        assert (mine[~fin] == theirs[~fin]).all() or np.isnan(theirs[~fin]).all(), (case, name, "inf")
        # per view where the whole gradient is stored (a degenerate face of one view does not set the
        # scale of another), else the whole output's
        rows = ref.rows(name)
        view = rows // F if F else rows
        err = 0.0
        for b in np.unique(view):
            m = (view == b)[:, None] & fin
            scale = np.abs(theirs[m]).max() if m.any() else 0.0
            if "rows" in ref.e[name]:
                scale = ref.scale(name)
            if m.any() and scale > 0:
                err = max(err, float(np.abs(mine[m] - theirs[m]).max() / scale))
        print(f"[{case} D={D}] {name}: {err:.2e} of scale, entries {int((idx >= 0).sum())}")
        assert err <= SAME, (case, name, err)
