"""Every soft-mask kernel path against the oracle.

The launcher picks the soft-mask kernels from knum, the size of the hit cache and whether the
backward finds the forward's state in the workspace (dibr_b200.cu: launch_fwd, backward_impl):

  forward   soft_fwd_kernel + soft_tiles_fwd_kernel<leftovers>   knum <= kSoftFwdK, a cache block or more
            soft_tiles_fwd_kernel (caching while blocks last)     knum > kSoftFwdK, or no cache block
            soft_tiles_fwd_kernel (K-lists)                       the operator dibr_soft_mask_forward_cuda
  backward  soft_bwd_runs_kernel + <leftovers>                    BINS_VALID, the forward used cache blocks
            dibr_tile_soft_bwd_kernel<leftovers>                  BINS_VALID, no cache block
            dibr_tile_soft_bwd_kernel<all tiles>                  no forward state (fresh workspace)
            soft_bwd_lists_kernel                                 the operator dibr_soft_mask_backward_cuda

Each case asserts through the per-launch trace which of them ran, at knum in {1, 30, 32, 33, 100} and
with no, a partial and a full hit cache (set through dibr_b200_workspace_bytes_cached).  The scenes
reach the work-list and window branches inside the kernels: partial 16x16 tiles, pixels with more
than knum candidates, tiles with more than kSoftCap (1024) candidates whose first index window is
empty, a view whose work list is the whole view (view_flag) with tiles that have no candidate at all,
an all-covered view, a view with no face near it, zero-area faces, and 1-pixel-high / -wide images.

Forward: the soft mask is within 1e-6 of the oracle and bit-identical across every cache size and
entry point (the fold is the reference's loop term for term in every path); the K-lists have the
oracle's face indices and dist_types exactly, its probabilities within 1e-6 and the reference's
padding.  Backward: every path within 3e-5 of the double-accumulating oracle and within 1e-6 of
the recompute over all tiles (they differ in the order of the float atomics, and the runs kernel
multiplies by 1/multiplier where the others divide), for three (multiplier, sigmainv) pairs.
"""
import collections
import functools

import numpy as np
import pytest
import torch

import oracle
from kaolin_b200 import _C, _lib, synthetic
from kaolin_b200.render.mesh import _host, dibr_soft_mask

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SIGMAINV, BOXLEN, MULT, EPS = 7000., 0.02, 1000., 1e-8     # the public API's defaults
KNUMS = [1, 30, 32, 33, 100]
PARAMS = [(1000., 7000.), (100., 70.), (1., 7000.)]          # (multiplier, sigmainv)
CACHES = ["none", "partial", "full"]
SOFT_FWD_K = 32     # kSoftFwdK: largest knum of the fused forward
SOFT_CAP = 1024     # kSoftCap: candidates one index window may hold
TILE = 16
TOL = 3e-5          # against the double-accumulating oracle, of the gradient's scale (test_parity_gpu.py)
SAME = 1e-6         # the same sums in another order of the float atomics
# except on the 520 x 520 scene, where a face collects thousands of terms: soft_bwd_lists_kernel adds
# every (pixel, face) term with a float atomic of its own, as the reference's kernel does, the runs
# kernel one per run of up to 8 cached hits of a face, while the recompute adds a tile's terms first.  The order alone put
# the lists kernel up to 2.4e-6 and the runs kernel up to 1.1e-6 of the gradient's scale from the
# recompute (measured on an H100, all three parameter pairs); every path stayed within 7e-7 of the
# oracle there.
SAME_BY_SCENE = {"whole_view": 5e-6}
PROB = 1e-6         # exp on the GPU and in the C library may round differently

FUSED, LEFT_FWD, SINGLE = "soft_fwd_kernel", "soft_tiles_fwd_kernel<leftovers>", "soft_tiles_fwd_kernel"
RUNS, LEFT_BWD = "soft_bwd_runs_kernel", "dibr_tile_soft_bwd_kernel<leftovers>"
ALL_TILES, LISTS = "dibr_tile_soft_bwd_kernel<all tiles>", "soft_bwd_lists_kernel"


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def npy(x):
    return x.detach().cpu().numpy()


def traced(fn, *args, **kw):
    """-> (fn's result, names of the soft-mask kernels it launched, in order)."""
    _lib.trace_begin()
    try:
        out = fn(*args, **kw)
    finally:
        ran = [name for name, _ in _lib.trace_end()]
    return out, [k for k in ran if "soft" in k]


def assert_grad_close(ours, ref, tol, what):
    """Max-normalised error <= tol AND element-wise allclose(rtol=tol, atol=tol * the gradient's scale)."""
    ours = npy(ours) if isinstance(ours, torch.Tensor) else ours
    ref = npy(ref) if isinstance(ref, torch.Tensor) else ref
    scale = max(float(np.abs(ref).max()), 1e-30)
    e = float(np.abs(ours - ref).max() / scale)
    assert e <= tol, (what, e)
    assert np.allclose(ours, ref, rtol=tol, atol=tol * scale), what


# ---------------------------------------------------------------------------------------------------
# the launcher's rules, restated
def soft_fwd_kernels(knum, cache_tiles):
    """launch_fwd: the fused kernel, then the single kernel over the tiles it could not cache, when
    knum <= kSoftFwdK and the workspace holds a cache block; else the single kernel alone."""
    return [FUSED, LEFT_FWD] if knum <= SOFT_FWD_K and cache_tiles > 0 else [SINGLE]


def soft_bwd_kernels(cache_tiles, bins_valid):
    """backward_impl: without the forward's bins every tile is recomputed; with them the runs
    kernel streams the cache blocks (if the workspace holds any) and the tiles the cache could not
    hold are recomputed."""
    if not bins_valid:
        return [ALL_TILES]
    return [RUNS, LEFT_BWD] if cache_tiles > 0 else [LEFT_BWD]


def pixel_rects(fvi, H, W, boxlen, multiplier):
    """(x_lo, x_hi, y_lo, y_hi) of every face: the pixels whose centre passes the reference's
    half-open test against the enlarged box [min - boxlen*m, max + boxlen*m) of the multiplied
    vertices (dibr_math.cuh: bbox_to_rect), as (B, F) int arrays."""
    m = np.float32(multiplier)
    v = np.asarray(fvi, np.float32) * m
    margin = np.float32(boxlen * multiplier)
    xmin, xmax = v[..., 0].min(-1) - margin, v[..., 0].max(-1) + margin
    ymin, ymax = v[..., 1].min(-1) - margin, v[..., 1].max(-1) + margin
    px = np.arange(1 - W, W, 2, dtype=np.int64).astype(np.float32) * (m / np.float32(W))     # ascending
    py = np.arange(H - 1, -H, -2, dtype=np.int64).astype(np.float32) * (m / np.float32(H))   # descending
    rising = py[::-1]
    x_lo, x_hi = np.searchsorted(px, xmin, "left"), np.searchsorted(px, xmax, "left")       # #{x0 < v}
    y_lo, y_hi = H - np.searchsorted(rising, ymax, "left"), H - np.searchsorted(rising, ymin, "left")  # #{y0 >= v}
    return x_lo, x_hi, y_lo, y_hi


def tile_spans(fvi, H, W, boxlen, multiplier):
    """-> (live, tx0, tx1, ty0, ty1): the 16x16 tiles each enlarged rectangle meets (live: not empty)."""
    x_lo, x_hi, y_lo, y_hi = pixel_rects(fvi, H, W, boxlen, multiplier)
    live = (x_hi > x_lo) & (y_hi > y_lo)
    return live, x_lo >> 4, (x_hi - 1) >> 4, y_lo >> 4, (y_hi - 1) >> 4


def sets_view_flag(fvi, H, W, boxlen, multiplier):
    """bin_faces_kernel: a view is flagged (its whole work list is every tile with an uncovered
    pixel) when one enlarged rectangle spans more than 64 (tile row x 32-tile word) cells."""
    live, tx0, tx1, ty0, ty1 = tile_spans(fvi, H, W, boxlen, multiplier)
    cells = (ty1 - ty0 + 1) * ((tx1 >> 5) - (tx0 >> 5) + 1)
    return (live & (cells > 64)).any(axis=1)


def tile_candidates(fvi, H, W, boxlen, multiplier):
    """(B, tiles_y, tiles_x) number of faces whose enlarged rectangle meets each 16x16 tile: the
    candidates soft_collect gathers for it."""
    B = fvi.shape[0]
    nty, ntx = -(-H // TILE), -(-W // TILE)
    live, tx0, tx1, ty0, ty1 = tile_spans(fvi, H, W, boxlen, multiplier)
    d = np.zeros((B, nty + 1, ntx + 1), np.int64)
    b = np.broadcast_to(np.arange(B)[:, None], live.shape)[live]
    tx0, tx1, ty0, ty1 = tx0[live], tx1[live] + 1, ty0[live], ty1[live] + 1
    for dy, dx, s in ((ty0, tx0, 1), (ty0, tx1, -1), (ty1, tx0, -1), (ty1, tx1, 1)):
        np.add.at(d, (b, dy, dx), s)
    return d.cumsum(1).cumsum(2)[:, :nty, :ntx]


def pixel_candidates(fvi, H, W, boxlen, multiplier):
    """(B, H, W) number of faces whose enlarged rectangle contains each pixel centre."""
    B = fvi.shape[0]
    x_lo, x_hi, y_lo, y_hi = pixel_rects(fvi, H, W, boxlen, multiplier)
    live = (x_hi > x_lo) & (y_hi > y_lo)
    d = np.zeros((B, H + 1, W + 1), np.int64)
    b = np.broadcast_to(np.arange(B)[:, None], live.shape)[live]
    x_lo, x_hi, y_lo, y_hi = x_lo[live], x_hi[live], y_lo[live], y_hi[live]
    for dy, dx, s in ((y_lo, x_lo, 1), (y_lo, x_hi, -1), (y_hi, x_lo, -1), (y_hi, x_hi, 1)):
        np.add.at(d, (b, dy, dx), s)
    return d.cumsum(1).cumsum(2)[:, :H, :W]


def uncovered_tiles(idx):
    """(B, tiles_y, tiles_x): the tile has a pixel no face covers."""
    B, H, W = idx.shape
    nty, ntx = -(-H // TILE), -(-W // TILE)
    pad = np.zeros((B, nty * TILE, ntx * TILE), bool)
    pad[:, :H, :W] = idx < 0
    return pad.reshape(B, nty, TILE, ntx, TILE).any(axis=(2, 4))


def hit_tiles(fvi, idx, boxlen, multiplier):
    """Tiles that claim a hit-cache block: filed in the work list (an uncovered pixel under some
    enlarged rectangle, counted per tile or through view_flag) with at least one candidate."""
    H, W = idx.shape[1:]
    return int((uncovered_tiles(idx) & (tile_candidates(fvi, H, W, boxlen, multiplier) > 0)).sum())


def first_window(n, F):
    """soft_window's first index window (-1, hi] for a tile with n > kSoftCap candidates out of F
    faces: a width guessed from the average index density."""
    return max(F * SOFT_CAP * 3 // (n * 4), 1) - 1


# ---------------------------------------------------------------------------------------------------
# scenes: (B, F, 3, 2) vertices in [-1, 1], 2-3 views each
Scene = collections.namedtuple("Scene", "fvz fvi fnz H W")


def offscreen(n, rng):
    """n small front-facing faces far right of the image: no enlarged rectangle reaches a pixel."""
    fvi = (np.array([5.0, 0.0]) + rng.normal(scale=0.05, size=(n, 3, 2))).astype(np.float32)
    return rng.uniform(-3, -1, size=(n, 3)).astype(np.float32), fvi, np.ones(n, np.float32)


def cluster(n, centre, rng):
    """n sub-pixel front-facing triangles (at 64 px) over the middle of the tile around `centre`."""
    c = np.asarray(centre) + rng.uniform(-0.1, 0.1, size=(n, 1, 2))
    fvi = (c + rng.normal(scale=0.004, size=(n, 3, 2))).astype(np.float32)
    return rng.uniform(-3, -1, size=(n, 3)).astype(np.float32), fvi, np.ones(n, np.float32)


def stack(*views):
    """Views given as lists of (fvz, fvi, fnz) parts -> (B, F, ...) arrays."""
    return tuple(np.stack([np.concatenate([p[i] for p in parts]) for parts in views]) for i in range(3))


def scene_mesh():
    """Icosphere views close enough to the camera that the silhouette crosses the image border, at
    a size that is not a multiple of 16 either way: partial tiles with hits."""
    return Scene(*synthetic.icosphere_views(3, 3, seed=71, radius=2.3), 200, 184)


def scene_soup():
    """Overlapping soup of mostly back-facing faces (not rasterized, still soft-mask candidates):
    nearly every uncovered pixel has more than 33 candidates, a third of them more than 100."""
    fvz, fvi, fnz = synthetic.triangle_soup(2, 2000, seed=72, coverage=150.0)
    fnz = np.where(np.random.default_rng(84).uniform(size=fnz.shape) < 0.03, 1.0, -1.0).astype(np.float32)
    return Scene(fvz, fvi, fnz, 72, 90)


def scene_windowed():
    """View 0: 2000 faces on the left half, then two clusters of 1100 sub-pixel triangles, each over
    one tile: more than kSoftCap candidates.  The first cluster's first index window holds part of
    it, the second's holds none of it.  View 1: as many faces spread over the image, no tile with
    more than kSoftCap candidates."""
    rng = np.random.default_rng(73)
    z, xy, n = synthetic.triangle_soup(1, 2000, seed=74, coverage=1.0)
    left = (z[0], (xy[0] * np.float32(0.4) - np.float32(0.5)).astype(np.float32), n[0])
    return Scene(*stack([left, cluster(1100, (0.75, -0.75), rng), cluster(1100, (0.75, 0.75), rng)],
                        [tuple(a[0] for a in synthetic.triangle_soup(1, 4200, seed=75, coverage=1.0))]), 64, 64)


def scene_whole_view():
    """View 0: two faces cover x > -0.2 of a 520 x 520 image.  Each one's enlarged rectangle spans all
    33 tile rows and both 32-tile words (it crosses column 512), so the view is flagged and every
    tile with an uncovered pixel is filed: the 5-pixel band left of the pair, which only the flag
    files, and the tiles further left, which no face is near.  View 1: an ordinary mesh."""
    rng = np.random.default_rng(76)
    pair = np.array([[[-0.2, -1.2], [1.2, -1.2], [1.2, 1.2]], [[-0.2, -1.2], [1.2, 1.2], [-0.2, 1.2]]], np.float32)
    z, xy, n = offscreen(78, rng)
    mesh = synthetic.icosphere_views(1, 1, seed=77)
    return Scene(*stack([(z[:40], xy[:40], n[:40]), (np.full((2, 3), -2.0, np.float32), pair, np.ones(2, np.float32)),
                         (z[40:], xy[40:], n[40:])], [tuple(a[0] for a in mesh)]), 520, 520)


def scene_edges():
    """View 0: two faces cover every pixel (empty work list).  View 1: no face near the image (the
    soft mask stays 0).  View 2: a soup with zero-area faces (three coincident vertices) and
    segments (two coincident vertices)."""
    rng = np.random.default_rng(78)
    quad = np.array([[[-1.5, -1.5], [1.5, -1.5], [1.5, 1.5]], [[-1.5, -1.5], [1.5, 1.5], [-1.5, 1.5]]], np.float32)
    cover = (np.full((2, 3), -2.0, np.float32), quad, np.ones(2, np.float32))
    z, xy, n = synthetic.triangle_soup(1, 20, seed=79, coverage=1.0)
    pts = rng.uniform(-0.9, 0.9, size=(10, 1, 2)).astype(np.float32).repeat(3, 1)
    seg = rng.uniform(-0.9, 0.9, size=(10, 3, 2)).astype(np.float32)
    seg[:, 2] = seg[:, 0]
    degenerate = (rng.uniform(-3, -1, size=(20, 3)).astype(np.float32), np.concatenate([pts, seg]),
                  np.where(rng.uniform(size=20) < 0.5, 1.0, -1.0).astype(np.float32))
    return Scene(*stack([cover, offscreen(38, rng)], [offscreen(40, rng)],
                        [(z[0], xy[0], n[0]), degenerate]), 40, 56)


def scene_row():
    return Scene(*synthetic.triangle_soup(2, 40, seed=80, coverage=2.0), 1, 75)


def scene_column():
    return Scene(*synthetic.triangle_soup(2, 40, seed=81, coverage=2.0), 45, 1)


SCENES = {"mesh": scene_mesh, "soup": scene_soup, "windowed": scene_windowed, "whole_view": scene_whole_view,
          "edges": scene_edges, "row": scene_row, "column": scene_column}


@functools.lru_cache(maxsize=None)
def scene(name):
    return SCENES[name]()


@functools.lru_cache(maxsize=None)
def gpu_scene(name):
    sc = scene(name)
    B, F = sc.fvi.shape[:2]
    return t(sc.fvz), t(sc.fvi), t(sc.fnz), t(synthetic.random_features(B, F, 1, seed=82))


@functools.lru_cache(maxsize=None)
def oracle_face_idx(name, multiplier):
    sc = scene(name)
    _, idx = oracle.rasterize(sc.H, sc.W, sc.fvz, sc.fvi, np.zeros(sc.fvz.shape + (1,), np.float32),
                              valid_faces=sc.fnz >= 0, multiplier=multiplier)
    return idx


def operator_inputs(fvi, multiplier):
    """The reference's arguments of dibr_soft_mask_forward_cuda (dibr.py:32-39): the multiplied
    vertices and their enlarged boxes."""
    fvi_m = np.asarray(fvi, np.float32) * np.float32(multiplier)
    margin = np.float32(BOXLEN * multiplier)
    return fvi_m, np.concatenate([fvi_m.min(-2) - margin, fvi_m.max(-2) + margin], -1)


@functools.lru_cache(maxsize=2)
def oracle_forward(name, knum, multiplier, sigmainv, all_uncovered=False):
    """-> (soft, prob, cidx, ctype) of the oracle, on its own face_idx or on all -1."""
    sc = scene(name)
    idx = oracle_face_idx(name, multiplier)
    if all_uncovered:
        idx = np.full_like(idx, -1)
    fvi_m, bb = operator_inputs(sc.fvi, multiplier)
    return oracle.soft_mask_forward_op(fvi_m, bb, idx, sigmainv, knum, multiplier)


@functools.lru_cache(maxsize=None)
def grad_soft(name):
    """Random on most pixels, exactly zero on a block of them."""
    sc = scene(name)
    B = sc.fvi.shape[0]
    g = np.random.default_rng(83).uniform(size=(B, sc.H, sc.W)).astype(np.float32)
    g[:, :max(1, sc.H // 2), :max(1, sc.W // 3)] = 0.
    return g


def cache_tiles(name, multiplier, cache):
    """Cache blocks for `cache`: none, about a third of the tiles that claim one, or every tile."""
    sc = scene(name)
    B = sc.fvi.shape[0]
    if cache == "none":
        return 0
    if cache == "full":
        return B * -(-sc.H // TILE) * -(-sc.W // TILE)
    hits = hit_tiles(sc.fvi, oracle_face_idx(name, multiplier), BOXLEN, multiplier)
    assert hits >= 2, (name, hits)
    return max(1, hits // 3)


# ---------------------------------------------------------------------------------------------------
# the C ABI
def forward(name, knum, multiplier, sigmainv, n_cache, face_idx_in=None):
    """dibr_b200_forward with a workspace holding `n_cache` hit-cache blocks: RASTER | SOFT_MASK, or
    SOFT_MASK alone on `face_idx_in`.  -> (face_idx, soft_mask, workspace)."""
    sc = scene(name)
    fvz, fvi, fnz, ff = gpu_scene(name)
    B, F = fvi.shape[:2]
    H, W = sc.H, sc.W
    raster = face_idx_in is None
    soft = torch.empty((B, H, W), dtype=torch.float32, device=DEV)
    idx = torch.empty((B, H, W), dtype=torch.int64, device=DEV) if raster else face_idx_in
    feat = torch.empty((B, H, W, 1), dtype=torch.float32, device=DEV) if raster else None
    n = _lib.lib().dibr_b200_workspace_bytes_cached(B, B * F, H, W, knum, n_cache)
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)
    p = _host.ptr
    st = _lib.lib().dibr_b200_forward(
        B, F, H, W, 1 if raster else 0, p(fvz) if raster else None, p(fvi), p(ff) if raster else None,
        p(fnz) if raster else None, None, multiplier, EPS, (_lib.RASTER if raster else 0) | _lib.SOFT_MASK,
        sigmainv, BOXLEN * multiplier, knum, p(feat), p(idx), None, p(soft), p(ws), n, _host.stream_ptr(DEV))
    _lib.check(st, "dibr_b200_forward")
    return idx, soft, ws


def backward(name, knum, multiplier, sigmainv, g_soft, idx, soft, ws):
    """dibr_b200_backward of the soft-mask branch alone: with the forward's workspace (BINS_VALID), or
    with ws=None on a fresh minimum-size workspace and no flag."""
    sc = scene(name)
    _, fvi, _, _ = gpu_scene(name)
    B, F = fvi.shape[:2]
    bins_valid = ws is not None
    if ws is None:
        ws = torch.empty(_lib.lib().dibr_b200_workspace_bytes(B, B * F, sc.H, sc.W), dtype=torch.uint8, device=DEV)
    g = torch.empty_like(fvi)
    p = _host.ptr
    st = _lib.lib().dibr_b200_backward(
        B, F, sc.H, sc.W, 0, None, p(g_soft), p(idx), None, p(soft), p(fvi), None, multiplier, EPS, sigmainv,
        BOXLEN * multiplier, knum, p(g), None, p(ws), ws.numel(), _lib.BINS_VALID if bins_valid else 0,
        _host.stream_ptr(DEV))
    _lib.check(st, "dibr_b200_backward")
    return g


def operator_forward(name, knum, multiplier, sigmainv, idx):
    fvi_m, bb = operator_inputs(scene(name).fvi, multiplier)
    return _C.render.mesh.dibr_soft_mask_forward_cuda(t(fvi_m), t(bb), idx, sigmainv, knum, multiplier)


# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SCENES))
def test_scene_reaches_its_branches(name):
    """Each scene has the property the module docstring gives it (host restatements of the binning)."""
    sc = scene(name)
    B, F = sc.fvi.shape[:2]
    idx = oracle_face_idx(name, MULT)
    cand = tile_candidates(sc.fvi, sc.H, sc.W, BOXLEN, MULT)
    flag = sets_view_flag(sc.fvi, sc.H, sc.W, BOXLEN, MULT)
    filed = uncovered_tiles(idx) & ((cand > 0) | flag[:, None, None])
    assert filed.any()
    assert flag.tolist() == [name == "whole_view"] + [False] * (B - 1)
    if name == "mesh":
        assert sc.H % TILE and sc.W % TILE and filed[:, -1, :].any() and filed[:, :, -1].any()
    if name == "soup":
        many = pixel_candidates(sc.fvi, sc.H, sc.W, BOXLEN, MULT)[idx < 0]
        assert (many > 100).mean() > 0.3 and (many > 33).mean() > 0.9, ((many > 100).mean(), (many > 33).mean())
    if name == "windowed":
        assert cand[1].max() <= SOFT_CAP
        big = [(ty, tx) for ty, tx in zip(*np.nonzero(cand[0] > SOFT_CAP))]
        assert len(big) == 2 and all(filed[0][c] for c in big)
        live, tx0, tx1, ty0, ty1 = tile_spans(sc.fvi[:1], sc.H, sc.W, BOXLEN, MULT)
        in_first = []
        for ty, tx in big:
            meets = np.nonzero(live[0] & (tx0[0] <= tx) & (tx <= tx1[0]) & (ty0[0] <= ty) & (ty <= ty1[0]))[0]
            in_first.append(int((meets <= first_window(len(meets), F)).sum()))
        assert sorted(in_first)[0] == 0 and 0 < sorted(in_first)[1] <= SOFT_CAP, in_first
    if name == "whole_view":
        assert (filed[0] & (cand[0] == 0)).any()      # filed through view_flag alone: no candidate
    if name == "edges":
        assert (idx[0] >= 0).all() and not filed[1].any() and filed[2].any()
    if name in ("row", "column"):
        assert min(sc.H, sc.W) == 1 and filed.sum() >= 2


@pytest.mark.parametrize("knum", KNUMS)
@pytest.mark.parametrize("name", list(SCENES))
def test_forward(name, knum):
    m, sig = MULT, SIGMAINV
    _, fvi, _, _ = gpu_scene(name)
    o_idx = oracle_face_idx(name, m)
    o_soft, o_prob, o_cidx, o_ctype = oracle_forward(name, knum, m, sig)
    t_idx = t(o_idx)
    softs = {}
    for cache in CACHES:
        n = cache_tiles(name, m, cache)
        (idx, soft, _), ran = traced(forward, name, knum, m, sig, n)
        assert ran == soft_fwd_kernels(knum, n), (cache, ran)
        assert np.array_equal(npy(idx), o_idx)
        softs["RASTER|SOFT_MASK", cache] = soft
        (_, soft, _), ran = traced(forward, name, knum, m, sig, n, face_idx_in=t_idx)
        assert ran == soft_fwd_kernels(knum, n), (cache, ran)
        softs["SOFT_MASK", cache] = soft
    softs["dibr_soft_mask"] = dibr_soft_mask(fvi, t_idx, sig, BOXLEN, knum, m)
    (k_soft, prob, cidx, ctype), ran = traced(operator_forward, name, knum, m, sig, t_idx)
    assert ran == [SINGLE], ran
    np.testing.assert_allclose(npy(k_soft), o_soft, rtol=0, atol=1e-6)
    for path, soft in softs.items():
        assert torch.equal(soft, k_soft), path

    cidx, ctype, prob = npy(cidx), npy(ctype), npy(prob)
    assert np.array_equal(cidx, o_cidx)
    assert np.array_equal(ctype, o_ctype)
    np.testing.assert_allclose(prob, o_prob, rtol=0, atol=PROB)
    hits = (cidx >= 0).sum(-1, keepdims=True)
    pad = np.arange(knum) >= hits
    assert (cidx[~pad] >= 0).all() and (ctype[~pad] >= 1).all() and (ctype[~pad] <= 6).all()
    assert (cidx[pad] == -1).all() and (prob[pad] == 0).all() and (ctype[pad] == 0).all()
    assert (hits[o_idx >= 0] == 0).all()

    # a user selected_face_idx of all -1: every pixel uncovered
    none = torch.full_like(t_idx, -1)
    u_soft = dibr_soft_mask(fvi, none, sig, BOXLEN, knum, m)
    uk_soft, u_prob, u_cidx, u_ctype = operator_forward(name, knum, m, sig, none)
    assert torch.equal(u_soft, uk_soft)
    o_u = oracle_forward(name, knum, m, sig, all_uncovered=True)
    np.testing.assert_allclose(npy(u_soft), o_u[0], rtol=0, atol=1e-6)
    assert np.array_equal(npy(u_cidx), o_u[2]) and np.array_equal(npy(u_ctype), o_u[3])
    np.testing.assert_allclose(npy(u_prob), o_u[1], rtol=0, atol=PROB)


@pytest.mark.parametrize("m,sig", PARAMS, ids=[f"m{m:g}-s{s:g}" for m, s in PARAMS])
@pytest.mark.parametrize("knum", KNUMS)
@pytest.mark.parametrize("name", list(SCENES))
def test_backward(name, knum, m, sig):
    o_idx = oracle_face_idx(name, m)
    o_soft, _, o_cidx, o_ctype = oracle_forward(name, knum, m, sig)
    g_soft = t(grad_soft(name))
    fvi_m, _ = operator_inputs(scene(name).fvi, m)

    grads = {}
    for cache in CACHES:
        n = cache_tiles(name, m, cache)
        idx, soft, ws = forward(name, knum, m, sig, n)
        assert np.array_equal(npy(idx), o_idx)
        np.testing.assert_allclose(npy(soft), o_soft, rtol=0, atol=1e-6)
        grads[cache], ran = traced(backward, name, knum, m, sig, g_soft, idx, soft, ws)
        assert ran == soft_bwd_kernels(n, True), (cache, ran)
    grads["all tiles"], ran = traced(backward, name, knum, m, sig, g_soft, idx, soft, None)
    assert ran == soft_bwd_kernels(0, False), ran

    k_soft, prob, cidx, ctype = operator_forward(name, knum, m, sig, idx)
    assert torch.equal(k_soft, soft)
    assert np.array_equal(npy(cidx), o_cidx) and np.array_equal(npy(ctype), o_ctype)
    grads["lists"], ran = traced(_C.render.mesh.dibr_soft_mask_backward_cuda, g_soft, k_soft, idx, prob, cidx,
                                 ctype, t(fvi_m), sig, m)
    assert ran == [LISTS], ran

    # The oracle differentiates the soft mask and probabilities the forward computed.  Where the soft
    # mask is 1 - 6e-8 the factor (1 - soft) of every term is one ulp: the ulp by which expf on the
    # GPU and in the C library may differ (PROB) moved a gradient entry by 8e-5 of the gradient's
    # scale (windowed scene, knum 30) when the oracle used its own forward.
    o_g = oracle.soft_mask_backward_op(npy(g_soft), npy(soft), o_idx, npy(prob), o_cidx, o_ctype, fvi_m, sig, m)
    for path, g in grads.items():
        assert_grad_close(g, o_g, TOL, path)
        assert_grad_close(g, grads["all tiles"], SAME_BY_SCENE.get(name, SAME), path)
