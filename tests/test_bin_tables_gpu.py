"""The bin tables the forward leaves in its workspace, compared exactly with the host restatement of the
binning (pixel_rects, bin_span and levels_for of test_binning_matrix_gpu.py).

After a forward (and after a backward that rebuilds the enlarged set without the forward's bins; it
takes no depth, so there only a NaN in face_vertices_image taints a face) the workspace holds, per
(set, view): the counters (entries per bin), their exclusive scan `off`, and the bin entries {face, x_lo | x_hi << 16, y_lo | y_hi << 16, 0} at off[bin] in the (set, view) region;
and per view the soft-mask tile bitmask (one bit per 16x16 tile under a live enlarged rectangle of at
most 64 (tile row, 32-tile word) cells) and view_flag (a larger one exists).  The order of the entries
inside a bin is unspecified, so each bin is compared sorted by face.  Sets the call does not bin have
zero counters.

Sparse meshes whose view's counters fit in shared memory are counted by bin_count_chunk_kernel
(view-owned chunks of 256..2048 faces) and filled by bin_fill_chunk_kernel (view-owned chunks of 256
faces); dense meshes take the aggregating bin_faces_kernel and the rest (large images) the plain one.
The kernels that ran are read from torch.profiler: the launch trace names the stage, not the kernel
behind it.  Scenes: the c4_shard, c3 and c2 benchmark scenes at full size; the
binning-matrix shapes on either side of a change of the number of levels; views split by chunk
borders, and views smaller than one chunk; NaN-tainted, culled and invalid faces; sets 1, 2 and 3;
the float64 entry, whose float scene (scaled vertices, conservative boxes, validity) is read from the
same workspace; and shapes that take the two fallbacks.
"""
import ctypes
import functools
import os
import subprocess

import numpy as np
import pytest
import torch

import test_binning_matrix_gpu as bm
import test_workspace_layout_cpu as wlc
from kaolin_b200 import _lib, synthetic
from kaolin_b200.render.mesh import _host

DEV = "cuda"
SIGMAINV, EPS, MULT = 7000., 1e-8, 1000.
CHUNK_THREADS, CHUNK_MAX_PER_THREAD, CHUNK_TARGET_CTAS = 256, 8, 2 * 132
CHUNK_SMEM_BUDGET = 48 * 1024


@functools.lru_cache(maxsize=None)
def layout_lib():
    """tests/host_math/workspace_layout.cpp: the header's carve, compiled on the host."""
    if not os.path.exists(wlc.LIB) or os.path.getmtime(wlc.LIB) < max(os.path.getmtime(wlc.SRC), os.path.getmtime(wlc.HDR)):
        os.makedirs(os.path.dirname(wlc.LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", wlc.LIB, wlc.SRC])
    lib = ctypes.CDLL(wlc.LIB)
    lib.wl_carve.argtypes = [ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                             ctypes.c_uint64, ctypes.c_uint64, ctypes.c_int64, ctypes.POINTER(ctypes.c_int64)]
    return lib


def piece(ws, d, name, dtype):
    at, nbytes = d[name]
    o = d["origin"] + at
    return ws[o:o + nbytes].view(dtype).cpu().numpy()


def geometry(H, W):
    L = bm.levels_for(H, W)
    ntx = np.array([bm.tiles(H, W, l)[0] for l in range(L)])
    nty = np.array([bm.tiles(H, W, l)[1] for l in range(L)])
    base = np.concatenate([[0], np.cumsum(ntx * nty)])
    return L, ntx, nty, base[:-1], int(base[-1])


def chunk_path(B, F, H, W, sets, first=False):
    """The launcher's choice: 'chunk' (with the chunk size), 'agg' or 'plain'."""
    _, ntx, nty, _, NB = geometry(H, W)
    if F >= 32 * ntx[0] * nty[0]:
        return "agg", None
    words = ((sets & 1) + (sets >> 1 & 1)) * NB + ((nty[0] * -(-ntx[0] // 32) + 1) if sets & 2 else 0)
    if first or 4 * words > CHUNK_SMEM_BUDGET:
        return "plain", None
    per = min(max(B * F // (CHUNK_TARGET_CTAS * CHUNK_THREADS), 1), CHUNK_MAX_PER_THREAD)
    return "chunk", CHUNK_THREADS * per


def box_rects(xmin, ymin, xmax, ymax, H, W, m):
    """bbox_to_rect of given float boxes (the float64 path's conservative ones)."""
    mf = np.float32(m)
    px = np.arange(1 - W, W, 2).astype(np.float32) * (mf / np.float32(W))
    rising = (np.arange(H - 1, -H, -2).astype(np.float32) * (mf / np.float32(H)))[::-1]
    return (np.searchsorted(px, xmin, "left"), np.searchsorted(px, xmax, "left"),
            H - np.searchsorted(rising, ymax, "left"), H - np.searchsorted(rising, ymin, "left"))


def expected_table(rect, has, H, W):
    """-> (counts (B, NB), rows (view, bin, face, x packed, y packed) sorted)."""
    L, ntx, _, base, NB = geometry(H, W)
    h, lvl, bx0, bx1, by0, by1 = bm.bin_span(tuple(np.asarray(r, np.int64) for r in rect), has, L)
    B = h.shape[0]
    x_lo, x_hi, y_lo, y_hi = (np.asarray(r, np.int64) for r in rect)
    rows = []
    for dy in (0, 1):
        for dx in (0, 1):
            bx, by = bx0 + dx, by0 + dy
            on = h & (bx <= bx1) & (by <= by1)
            v, f = np.nonzero(on)
            l = lvl[on]
            rows.append(np.stack([v, base[l] + by[on] * ntx[l] + bx[on], f,
                                  x_lo[on] | (x_hi[on] << 16), y_lo[on] | (y_hi[on] << 16)], 1))
    rows = np.concatenate(rows)
    counts = np.zeros((B, NB), np.int64)
    np.add.at(counts, (rows[:, 0], rows[:, 1]), 1)
    return counts, rows[np.lexsort(rows.T[::-1])]


def expected_bitmask(rect, live, H, W):
    """-> ((B, nty, words) uint32 tile bitmask, (B,) view_flag)."""
    x_lo, x_hi, y_lo, y_hi = (np.asarray(r, np.int64) for r in rect)
    flag, cells = bm.view_flags(rect, live, H, W)
    ntx, nty = bm.tiles(H, W)
    nw = -(-ntx // 32)
    on = (cells > 0) & (cells <= 64)
    v, f = np.nonzero(on)
    tx0, tx1 = x_lo[on] >> 4, (x_hi[on] - 1) >> 4
    ty0, ty1 = y_lo[on] >> 4, (y_hi[on] - 1) >> 4
    diff = np.zeros((len(flag), nty + 1, ntx + 1), np.int64)
    for yy, xx, s in ((ty0, tx0, 1), (ty0, tx1 + 1, -1), (ty1 + 1, tx0, -1), (ty1 + 1, tx1 + 1, 1)):
        np.add.at(diff, (v, yy, xx), s)
    cov = diff.cumsum(1).cumsum(2)[:, :nty, :ntx] > 0
    cov = np.concatenate([cov, np.zeros((len(flag), nty, nw * 32 - ntx), bool)], 2).reshape(len(flag), nty, nw, 32)
    words = (cov.astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(-1).astype(np.uint32)
    return words, flag


def check_tables(ws, shape, F, H, W, sets, rects, has, live):
    """Compares the workspace's tables with the host restatement: rects[set] and has[set] per set,
    live (the enlarged set's rule) for the bitmask."""
    B = shape[0]
    out = (ctypes.c_int64 * 64)()
    layout_lib().wl_carve(*shape, ws.data_ptr(), ws.numel(), shape[1], out)
    r = list(out)
    d = dict(zip(["fits", "origin"], r[:2]))
    for i, name in enumerate(wlc.NAMES):
        d[name] = (r[6 + 2 * i], r[7 + 2 * i])
    assert d["fits"]
    _, _, _, _, NB = geometry(H, W)
    cnt = piece(ws, d, "cnt", torch.int32).reshape(2, B, NB).astype(np.int64)
    off = piece(ws, d, "off", torch.int32).reshape(2, B, NB).astype(np.int64)
    ent = piece(ws, d, "entries", torch.int32).reshape(2, -1, 4)
    for st in (0, 1):
        if not (sets >> st) & 1:
            assert not cnt[st].any(), st
            continue
        want_cnt, want_rows = expected_table(rects[st], has[st], H, W)
        assert np.array_equal(cnt[st], want_cnt), (st, np.argwhere(cnt[st] != want_cnt)[:8])
        excl = np.concatenate([np.zeros((B, 1), np.int64), np.cumsum(want_cnt, 1)[:, :-1]], 1)
        assert np.array_equal(off[st], excl), st
        got = []
        for b in range(B):
            n = int(want_cnt[b].sum())
            e = ent[st, 4 * b * F: 4 * b * F + n].astype(np.int64)
            assert (e[:, 3] == 0).all()
            binid = np.repeat(np.arange(NB), want_cnt[b])
            got.append(np.stack([np.full(n, b), binid, e[:, 0], e[:, 1], e[:, 2]], 1))
        got = np.concatenate(got)
        got = got[np.lexsort(got.T[::-1])]
        assert np.array_equal(got, want_rows), (st, len(got), len(want_rows))
    if sets & 2:
        words, flag = expected_bitmask(rects[1], live, H, W)
        got_words = piece(ws, d, "tile_cnt", torch.int32).view(np.uint32)[:words.size].reshape(words.shape)
        assert np.array_equal(got_words, words)
        assert np.array_equal(piece(ws, d, "view_flag", torch.int32)[:B] != 0, flag)
    return d


def profiled(fn):
    """-> (result, names of the bin kernels that ran).  The tracer can drop the events of a profile,
    so a call whose profile shows no bin kernel is repeated (the tables do not depend on the run)."""
    from torch.profiler import ProfilerActivity, profile
    kinds = ("bin_count_chunk_kernel", "bin_fill_chunk_kernel", "bin_faces_kernel<false, false>", "bin_faces_kernel<true, false>",
             "bin_faces_kernel<false, true>", "bin_faces_kernel<true, true>")
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.ones(1, device=DEV).add_(1)     # the tracer can miss the first launch of a profile
            torch.cuda.synchronize()
            out = fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events()}
        ran = {k for k in kinds if any(k in n for n in names)}
        if ran:
            break
    return out, ran


def kernels_of(path):
    return {"chunk": {"bin_count_chunk_kernel", "bin_fill_chunk_kernel"},
            "plain": {"bin_faces_kernel<false, false>", "bin_faces_kernel<true, false>"},
            "agg": {"bin_faces_kernel<false, true>", "bin_faces_kernel<true, true>"}}[path]


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ---------------------------------------------------------------------------------------------------
# scenes: (fvz, fvi, fnz, valid_u8 or None, H, W, m, boxlen)
def bench_scene(B, level, H, W):
    fvz, fvi, fnz = synthetic.icosphere_views(B, level, seed=1234, jitter=0.05)
    return fvz, fvi, fnz, None, H, W, MULT, 0.02


def matrix_scene(name):
    sc = bm.scene(name)
    return sc.fvz, sc.fvi, sc.fnz, None, sc.H, sc.W, sc.m, sc.boxlen


def soup(B, F, H, W, seed, size=12.0):
    """Small random triangles over the image (and a little beyond it)."""
    rng = np.random.default_rng(seed)
    c = rng.uniform(-1.05, 1.05, size=(B, F, 1, 2))
    fvi = (c + rng.uniform(-size, size, size=(B, F, 3, 2)) / np.array([W, H])).astype(np.float32)
    fvz = rng.uniform(-3, -1, size=(B, F, 3)).astype(np.float32)
    fnz = rng.uniform(-0.2, 1, size=(B, F)).astype(np.float32)
    return fvz, fvi, fnz, None, H, W, MULT, 0.02


def tainted(B, F, H, W, seed):
    """A soup with NaN in one of the nine coordinates of 2 % of the faces, culled faces (fnz < 0)
    and invalid ones (valid_faces == 0)."""
    fvz, fvi, fnz, _, H, W, m, boxlen = soup(B, F, H, W, seed)
    rng = np.random.default_rng(seed + 1)
    bad = rng.uniform(size=(B, F)) < 0.02
    b, f = np.nonzero(bad)
    k = rng.integers(0, 9, len(b))
    z = k < 3
    fvz[b[z], f[z], k[z]] = np.nan
    fvi[b[~z], f[~z], (k[~z] - 3) // 2, (k[~z] - 3) % 2] = np.nan
    valid = (rng.uniform(size=(B, F)) > 0.1).astype(np.uint8)
    return fvz, fvi, fnz, valid, H, W, m, boxlen


SCENES = {
    "c4_shard": lambda: bench_scene(32, 5, 1024, 1024),
    "c3": lambda: bench_scene(64, 5, 512, 512),
    "c2": lambda: bench_scene(8, 4, 256, 256),
    **{f"levels_{H}x{W}": functools.partial(matrix_scene, f"levels_{H}x{W}")
       for H, W in ((17, 9), (64, 65), (65, 64), (256, 257), (1024, 1025))},
    "culled": functools.partial(matrix_scene, "culled"),
    "chunk_borders": lambda: soup(5, 70001, 1024, 1024, 7),     # 1280-face chunks, the last one partial
    "small_views": lambda: soup(3, 100, 200, 300, 8),            # one 256-face chunk, mostly empty
    "tainted": lambda: tainted(4, 30000, 512, 512, 9),
    # fallbacks: counters beyond the shared-memory budget (plain), a dense mesh (aggregating)
    "levels_4096x4097": functools.partial(matrix_scene, "levels_4096x4097"),
    "soup_2048": lambda: soup(2, 3000, 2048, 2048, 10, size=40.0),
    "mixed_warp": functools.partial(matrix_scene, "mixed_warp"),
}


PATHS = {"culled": "agg", "mixed_warp": "agg", "levels_4096x4097": "plain", "soup_2048": "plain"}   # else chunk


@functools.lru_cache(maxsize=None)
def scene(name):
    return SCENES[name]()


def host_rects(sc):
    fvz, fvi, fnz, valid, H, W, m, boxlen = sc
    live = ~(np.isnan(fvi).any((-1, -2)) | np.isnan(fvz).any(-1))
    ok = live & (fnz >= 0)
    if valid is not None:
        ok &= valid != 0
    return [bm.pixel_rects(fvi, H, W, m), bm.pixel_rects(fvi, H, W, m, boxlen * m)], [ok, live], live


def run_forward(sc, sets, knum=30):
    fvz, fvi, fnz, valid, H, W, m, boxlen = sc
    B, F = fnz.shape
    D = 3
    ff = T(synthetic.random_features(B, F, D, seed=3))
    mode = (_lib.RASTER if sets & 1 else 0) | (_lib.SOFT_MASK if sets & 2 else 0)
    idx_in = None if sets & 1 else torch.full((B, H, W), -1, dtype=torch.int64, device=DEV)
    args = (mode, H, W, T(fvz), T(fvi), ff, T(fnz), None if valid is None else T(valid), m, EPS, SIGMAINV,
            boxlen * m, knum if sets & 2 else 0)
    _lib.trace_begin()
    try:
        out, ran = profiled(lambda: _host.forward(*args, face_idx_in=idx_in))
    finally:
        trace = [k for k, _ in _lib.trace_end()]
    assert trace[:3] == ["bin_faces_kernel<count>", "scan_bins_kernel", "bin_faces_kernel<fill>"], trace
    return out, ran


CASES = [(n, s) for n in SCENES for s in ((1, 2, 3) if n in ("c2", "tainted", "chunk_borders", "levels_1024x1025")
                                          else (3,))]


@pytest.mark.gpu
@pytest.mark.parametrize("name,sets", CASES, ids=[f"{n}-sets{s}" for n, s in CASES])
def test_forward_bin_tables(name, sets):
    sc = scene(name)
    fvz, fvi, fnz, valid, H, W, m, boxlen = sc
    B, F = fnz.shape
    path, chunk = chunk_path(B, F, H, W, sets)
    assert path == PATHS.get(name, "chunk"), path
    if name == "chunk_borders":
        assert chunk == 1280 and F % chunk and F > chunk
    if name == "small_views":
        assert F < chunk
    (_, _, _, _, ws), ran = run_forward(sc, sets)
    assert ran == kernels_of(path), (path, ran)
    rects, has, live = host_rects(sc)
    knum = 30 if sets & 2 else 0
    check_tables(ws, (B, B * F, H, W, knum, 0), F, H, W, sets, rects, has, live)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["c2", "tainted"])
def test_backward_rebuild_bin_tables(name):
    """A backward without the forward's bins rebuilds the enlarged set through the same launcher."""
    sc = scene(name)
    fvz, fvi, fnz, valid, H, W, m, boxlen = sc
    B, F = fnz.shape
    (_, idx, _, soft, ws), _ = run_forward(sc, 3)
    ff = T(synthetic.random_features(B, F, 3, seed=3))
    g_soft = T(np.random.default_rng(4).uniform(-1, 1, size=(B, H, W)).astype(np.float32))
    ws.zero_()
    _lib.trace_begin()
    try:
        _, ran = profiled(lambda: _host.backward(H, W, None, g_soft, idx, None, soft, T(fvi), ff, m, EPS, SIGMAINV,
                                                 boxlen * m, 30, ws, False))
    finally:
        trace = [k for k, _ in _lib.trace_end()]
    assert trace[:3] == ["bin_faces_kernel<count>", "scan_bins_kernel", "bin_faces_kernel<fill>"], trace
    assert ran == kernels_of(chunk_path(B, F, H, W, 2)[0])
    # the backward takes no depth: there a face is tainted by a NaN in face_vertices_image only
    rects, _, _ = host_rects(sc)
    live = ~np.isnan(fvi).any((-1, -2))
    check_tables(ws, (B, B * F, H, W, 30, 0), F, H, W, 2, rects, [None, live], live)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["c2", "tainted", "chunk_borders", "levels_4096x4097"])
def test_float64_bin_tables(name):
    """The float64 entry bins its float scene (scaled vertices, conservative boxes, validity) with the
    same kernels; that scene is read back from the workspace."""
    sc = scene(name)
    fvz, fvi, fnz, valid, H, W, m, boxlen = sc
    B, F = fnz.shape
    fvz64, fvi64 = fvz.astype(np.float64), fvi.astype(np.float64)
    ff = T(synthetic.random_features(B, F, 3, seed=3).astype(np.float64))
    args = (_lib.RASTER | _lib.SOFT_MASK, H, W, T(fvz64), T(fvi64), ff, T(fnz.astype(np.float64)),
            None if valid is None else T(valid), m, EPS, SIGMAINV, boxlen * m, 30)
    (_, _, _, _, ws), ran = profiled(lambda: _host.forward(*args))
    assert ran == kernels_of(chunk_path(B, F, H, W, 3)[0])
    out = (ctypes.c_int64 * 64)()
    shape = (B, B * F, H, W, 0, 1)
    layout_lib().wl_carve(*shape, ws.data_ptr(), ws.numel(), B * F, out)
    r = list(out)
    d = {"origin": r[1], **{n: (r[6 + 2 * i], r[7 + 2 * i]) for i, n in enumerate(wlc.NAMES)}}
    xy = piece(ws, d, "xy", torch.float32).reshape(B, F, 6)
    bt = piece(ws, d, "bbox_tight", torch.float32).reshape(B, F, 4)
    bl = piece(ws, d, "bbox_large", torch.float32).reshape(B, F, 4)
    ok = piece(ws, d, "valid", torch.uint8)[:B * F].reshape(B, F) != 0
    live = ~np.isnan(xy).any(-1)
    rects = [box_rects(*(b[..., k] for k in range(4)), H, W, m) for b in (bt, bl)]
    check_tables(ws, shape, F, H, W, 3, rects, [live & ok, live], live)
