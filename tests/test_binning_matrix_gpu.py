"""The float32 / bf16 rasterizer and soft mask against the reference's float kernels, bit for bit, on
images and scenes built to break the bin hierarchy.

Every float32 call bins its faces before any pixel is tested (dibr_b200.cu): bin_faces_kernel<count>,
scan_bins_kernel, bin_faces_kernel<fill>, then the tile consumers.  Each face's exact pixel rectangle
(bbox_to_rect, tight for the rasterizer and enlarged for the soft mask) goes to the finest level l at
which it spans at most 2x2 bins of 16 * 4^l px (bin_span), or to the coarsest level, whose one bin
holds the whole image (levels_for).  A rectangle off by one pixel, or one bin dropped, loses pixels:
unlike the float64 path the float32 path has no conservative superset to fall back on.  The host
restatement below (levels_for, bin_span, the aggregated / plain-atomics choice, the soft mask's tile
bitmask and its view_flag fallback) shows what each scene reaches:

  levels      (H, W) on both sides of every change of the number of levels (max(H, W) = 16 * 4^l + 1),
              with quads whose tight or enlarged rectangle has an edge on a bin boundary of its own
              level, or one pixel either side of it, and an image-wide and an image-high strip.
  promote     per level, quads spanning exactly 2x2 bins and exactly one bin (they stay) next to quads
              spanning 3 bins in one axis (they go one level up).
  max_dim     16384 x 16 and 16 x 16384 (6 levels, 1024 tiles and 32 bitmask words per row) and a
              64 x 16384 soup whose widest enlarged rectangles set view_flag.
  mixed_warp  a dense mesh (>= 32 faces per tile: the aggregating kernel) whose warps hold one
              image-sized face in lane 0, 15 or 31, all faces in one bin, or (16 warps over three CTAs)
              all faces in one hot bin.
  bitmask     W in {511, 512, 513, 1536}: enlarged rectangles ending on tile column 31 / 32 and on
              32-tile word boundaries, and spanning 64 (row x word) cells (per-tile bits) or 65 and 66
              (view_flag) in one view of a batch but not in its neighbour.
  culled      faces with face_normals_z < 0 (and a view of nothing else): the tight set skips them,
              the enlarged set still bins them for the soft mask.
  mult        multipliers 0.1, 333.3 and 1000: multiplier / W is rounded, pixel centres are off the
              binary lattice.

The aggregating kernel sends a warp to plain atomics when one of its faces spans more than 2x2 bins
at its level (__all_sync(small)).  bin_span only stops above 2x2 at the coarsest level, which is one
bin wide and high, so no warp takes that branch: the host model asserts it of every scene.

Bars: face_idx, features and soft mask digest-equal to the reference's for every scene, through
dibr_rasterization (knum 30: the fused soft-mask forward; knum 100: the single kernel), through
rasterize and dibr_soft_mask alone, and with D = 1.  bf16 features (the bars of
test_parity_gpu.py::test_bf16_feature_storage_vs_reference_cuda): face_idx and soft mask bit-equal,
the features the reference's float32 result on the bf16-rounded inputs rounded once to bf16, grad_ff
within 2^-8 of the reference's.  Gradients (float32 features): grad_fvi and grad_ff within 3e-5 of the
gradient's scale of the double-accumulating C oracle, and within the same bar of the reference's
gradients on its stored rows wherever the reference is within 1e-5 of the oracle.  Images of more
than ORACLE_MAX_PIXELS pixels (one levels case) are held to the reference's gradients alone, at that
bar: the C oracle walks every face for every pixel.  Reruns give byte-identical outputs.

NaN vertices, which make a face absent from every set, are held to the scene without them in
test_nan_vertices_gpu.py.
"""
import collections
import functools
import os

import numpy as np
import pytest
import torch

import oracle
from kaolin_b200 import _lib, synthetic
from oracle import ref_cuda, ref_golden

DEV = "cuda"
SIGMAINV, EPS = 7000., 1e-8
TILE = 16
KNUMS = (30, 100)
SOFT_FWD_K = 32              # kSoftFwdK: largest knum of the fused soft-mask forward
ROW_WALK_MAX_D, RW_SLAB = 4, 4
GRAD_TOL, REF_AGREES, BF16_TOL = 3e-5, 1e-5, 2.0 ** -8
ORACLE_MAX_PIXELS = 1 << 22
# the reference's outputs: digests of what is compared bit for bit, 64 sampled rows of each gradient
STORE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_cuda_binning.npz")
DIGEST_ONLY = ("face_idx", "features", "features_bf16", "soft_mask")

Case = collections.namedtuple("Case", "fvz fvi fnz H W m boxlen")


# ---------------------------------------------------------------------------------------------------
# the binning restated on the host
def levels_for(H, W):
    L = 1
    while (TILE << 2 * (L - 1)) < max(H, W):
        L += 1
    return L


def tiles(H, W, l=0):
    t = TILE << 2 * l
    return -(-W // t), -(-H // t)


def aggregating(B, F, H, W):
    """The launcher's choice of the aggregating bin kernel: >= 32 faces per finest bin on average."""
    ntx, nty = tiles(H, W)
    return (B * F) // B >= 32 * ntx * nty


def pixel_rects(fvi, H, W, m, margin=None):
    """bbox_to_rect of every face: [x_lo, x_hi) x [y_lo, y_hi), the pixels whose centre passes the
    half-open float test against the box of the multiplied vertices (enlarged by the float margin)."""
    mf = np.float32(m)
    v = np.asarray(fvi, np.float32) * mf
    xmin, xmax = v[..., 0].min(-1), v[..., 0].max(-1)
    ymin, ymax = v[..., 1].min(-1), v[..., 1].max(-1)
    if margin is not None:
        g = np.float32(margin)
        xmin, ymin, xmax, ymax = xmin - g, ymin - g, xmax + g, ymax + g
    px = np.arange(1 - W, W, 2).astype(np.float32) * (mf / np.float32(W))        # ascending
    rising = (np.arange(H - 1, -H, -2).astype(np.float32) * (mf / np.float32(H)))[::-1]
    return (np.searchsorted(px, xmin, "left"), np.searchsorted(px, xmax, "left"),
            H - np.searchsorted(rising, ymax, "left"), H - np.searchsorted(rising, ymin, "left"))


def bin_span(rect, has, L):
    """-> (has, level, bx0, bx1, by0, by1): the finest level at which the rectangle spans <= 2x2
    bins, else the coarsest; empty rectangles and faces the set skips have no bins."""
    x_lo, x_hi, y_lo, y_hi = rect
    has = has & (x_hi > x_lo) & (y_hi > y_lo)
    lvl = np.full(x_lo.shape, L - 1)
    for l in reversed(range(L - 1)):
        sh = 4 + 2 * l
        ok = (((x_hi - 1) >> sh) - (x_lo >> sh) <= 1) & (((y_hi - 1) >> sh) - (y_lo >> sh) <= 1)
        lvl = np.where(ok, l, lvl)
    lvl = np.where(has, lvl, 0)
    sh = 4 + 2 * lvl
    bx0, bx1 = np.where(has, x_lo >> sh, 0), np.where(has, (x_hi - 1) >> sh, -1)
    by0, by1 = np.where(has, y_lo >> sh, 0), np.where(has, (y_hi - 1) >> sh, -1)
    return has, lvl, bx0, bx1, by0, by1


def fallback_warps(span):
    """Warps (32 consecutive global face indices) of the aggregating kernel in which some face spans
    more than 2x2 bins at its level, so that __all_sync(small) sends the warp to plain atomics.  Lanes
    past the last face have no bins."""
    _, _, bx0, bx1, by0, by1 = (np.ravel(a) for a in span)
    small = (bx1 - bx0 <= 1) & (by1 - by0 <= 1)
    small = np.concatenate([small, np.ones(-len(small) % 32, bool)])
    return np.nonzero(~small.reshape(-1, 32).all(1))[0]


def view_flags(rect, live, H, W):
    """bin_faces_kernel's soft-mask tile bitmask: a live enlarged rectangle sets one bit per 16x16
    tile, a row of tiles per 32-tile word, unless it spans more than 64 (tile row x word) cells:
    then it flags its view.  -> ((B,) flag, (B, F) cells)."""
    x_lo, x_hi, y_lo, y_hi = rect
    live = live & (x_hi > x_lo) & (y_hi > y_lo)
    tx0, tx1, ty0, ty1 = x_lo >> 4, (x_hi - 1) >> 4, y_lo >> 4, (y_hi - 1) >> 4
    cells = np.where(live, (ty1 - ty0 + 1) * ((tx1 >> 5) - (tx0 >> 5) + 1), 0)
    return (cells > 64).any(1), cells


def analyse(sc, sets=3):
    """The host model's view of one call: rectangles, bin spans and the bin kernel per set."""
    B, F = sc.fnz.shape
    L = levels_for(sc.H, sc.W)
    tight = pixel_rects(sc.fvi, sc.H, sc.W, sc.m)
    large = pixel_rects(sc.fvi, sc.H, sc.W, sc.m, sc.boxlen * sc.m)
    valid = sc.fnz >= 0
    live = np.ones_like(valid)
    spans = [bin_span(tight, valid, L), bin_span(large, live, L)]
    flag, cells = view_flags(large, live, sc.H, sc.W)
    levels = [np.bincount(s[1][s[0]], minlength=L) for s in spans]
    return dict(L=L, tight=tight, large=large, spans=spans, flag=flag, cells=cells, levels=levels,
                agg=aggregating(B, F, sc.H, sc.W),
                fallback=[fallback_warps(spans[s]) for s in range(2) if (sets >> s) & 1])


# ---------------------------------------------------------------------------------------------------
# scenes, in the unscaled coordinates of face_vertices_image
def X(k, W):
    """x of the boundary between pixel columns k - 1 and k: midway between their centres."""
    return (2.0 * k - W) / W


def Y(k, H):
    return (H - 2.0 * k) / H


def quad(x0, x1, y0, y1, H, W, inset=0.0):
    """Two faces filling the pixel rectangle [x0, x1) x [y0, y1), their vertices on pixel boundaries;
    inset (in unscaled units, the boxlen) pulls the vertices in so that the ENLARGED rectangle is it."""
    a = (X(x0, W) + inset, Y(y0, H) - inset)
    b = (X(x1, W) - inset, Y(y0, H) - inset)
    c = (X(x0, W) + inset, Y(y1, H) + inset)
    d = (X(x1, W) - inset, Y(y1, H) + inset)
    return [[a, b, c], [b, d, c]]


def finish(views, H, W, m=1000., boxlen=0.02, seed=0, fnz=None):
    """views: per view a list of faces (3, 2) -> Case; depths differ per quad, so each face is flat."""
    rng = np.random.default_rng(seed)
    n = max(len(v) for v in views)
    fvi = np.zeros((len(views), n, 3, 2))
    fvi[..., 0] = 5.0                            # views with fewer faces are padded with faces off screen
    for b, v in enumerate(views):
        fvi[b, :len(v)] = v
    fvz = np.repeat(rng.uniform(-3, -1, size=(len(views), n, 1)), 3, axis=2)
    f = np.ones((len(views), n)) if fnz is None else fnz
    return Case(fvz.astype(np.float32), fvi.astype(np.float32), f.astype(np.float32), H, W, m, boxlen)


def edge_rects(H, W):
    """Per level below the coarsest, pixel rectangles of that level with one edge at k * 16 * 4^l + d,
    d in {-1, 0, 1}, on either side and along either axis -> [(x0, x1, y0, y1, inset)]: the tight
    rectangle is the target, or (inset) the enlarged one is."""
    out = []
    for l in range(levels_for(H, W) - 1):
        S = TILE << 2 * l
        w = 8 if l == 0 else S // 2 + 1          # more than 2 bins of level l - 1, at most 2 of level l
        for axis in (0, 1):
            n, other = (W, H) if axis == 0 else (H, W)
            for i, k in enumerate(sorted({k for k in (1, (n - 1) // S) if 0 < k * S < n})):
                for d in (-1, 0, 1):
                    for side in ("lo", "hi"):
                        for inset in (False, True):
                            e = k * S + d
                            a, b = (e, e + w) if side == "lo" else (e - w, e)
                            ext = min(other, 8 if inset else 4)
                            c = (7 * (i + 3 * d + 5) + 13 * l) % max(other - ext, 1)
                            if a < 0 or b > n or c + ext > other:
                                continue
                            out.append(((a, b, c, c + ext) if axis == 0 else (c, c + ext, a, b)) + (inset,))
    return out


def scene_levels(H, W):
    boxlen = 4.0 / max(H, W)                     # enlarged rectangles 2 px wider on a side, at most
    faces = []
    for x0, x1, y0, y1, inset in edge_rects(H, W):
        faces += quad(x0, x1, y0, y1, H, W, boxlen if inset else 0.0)
    faces += quad(0, W, H // 3, min(H // 3 + 2, H), H, W)            # image-wide and -high strips:
    faces += quad(W // 3, min(W // 3 + 2, W), 0, H, H, W)            # the coarsest level
    return finish([faces], H, W, boxlen=boxlen, seed=H * 7 + W)


def promote_rects(H, W):
    """(x0, x1, y0, y1, kind, level it must reach): per level l below the coarsest, rectangles of
    exactly 2x2 and 1x1 bins of level l, and of 3 bins in one axis (one level up)."""
    out = []
    for l in range(levels_for(H, W) - 1):
        S = TILE << 2 * l
        n = min(H, W) // S
        kinds = {"2x2": (2 * S, 2 * S, l), "1x1": (S, S, l), "3x": (2 * S + 1, S, l + 1), "3y": (S, 2 * S + 1, l + 1)}
        for kind, (ex, ey, to) in kinds.items():
            for k in range(min(3, n)):
                x0, y0 = k * S, ((2 * k + l + len(out)) % max(n - 2, 1)) * S
                if x0 + ex <= W and y0 + ey <= H:
                    out.append((x0, x0 + ex, y0, y0 + ey, kind, to))
    return out


def scene_promote():
    H = W = 1024
    faces = []
    for x0, x1, y0, y1, _, _ in promote_rects(H, W):
        faces += quad(x0, x1, y0, y1, H, W)
    return finish([faces], H, W, boxlen=0.004, seed=31)


def scene_soup_wide(H=64, W=16384, n=400, seed=32):
    """Triangles from 2 px to 12000 px wide and up to 24 px high, most of them small, and three wide ones."""
    rng = np.random.default_rng(seed)
    cx, cy = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    w = np.exp(rng.uniform(np.log(2.0), np.log(12000.0), n)) / W
    h = rng.uniform(1.0, 24.0, n) / H
    cx[:3], cy[:3], w[:3], h[:3] = 0.0, 0.0, 12000.0 / W, 1.0   # 12000 x 64 px: more than 64 (row x word) cells
    fvi = np.stack([np.stack([cx - w, cy - h], -1), np.stack([cx + w, cy - h * rng.uniform(-1, 1, n)], -1),
                    np.stack([cx + w * rng.uniform(-1, 1, n), cy + h], -1)], 1)
    return finish([list(fvi)], H, W, boxlen=0.0005, seed=seed)


def scene_mixed_warp():
    """B = 2 (the second view mirrored); 64 warps of 32 faces at 96 x 96 (36 tiles: >= 32 faces per tile)."""
    H = W = 96
    rng = np.random.default_rng(33)
    tiny = lambda cx, cy, n, s: (np.stack([cx, cy], -1)[:, None, :]
                                 + rng.uniform(-s, s, size=(n, 3, 2)))
    warps = []
    for wi in range(64):
        if wi < 48 and wi % 3 == 0:              # 16 warps, 2 kinds of CTAs: all in the hot bin (tile 2,2)
            warps.append(tiny(np.full(32, X(40, W)), np.full(32, Y(40, H)), 32, 0.06))
        elif wi % 4 == 1:                        # every face in one bin of the finest level
            tx, ty = rng.integers(0, 6, 2)
            warps.append(tiny(np.full(32, X(16 * tx + 8, W)), np.full(32, Y(16 * ty + 8, H)), 32, 0.05))
        else:                                    # scattered faces, one of them image-sized in lane 0, 15 or 31
            f = tiny(rng.uniform(-0.9, 0.9, 32), rng.uniform(-0.9, 0.9, 32), 32, 0.08)
            lane = (0, 15, 31, None)[(wi // 4) % 4]
            if lane is not None:
                f[lane] = [(-1.05, -1.05), (1.1, -1.02), (-1.03, 1.1)]
            warps.append(f)
    fvi = np.concatenate(warps)
    views = [list(fvi), list(fvi * np.array([-1.0, 1.0]))]
    sc = finish(views, H, W, boxlen=0.02, seed=34)
    z = sc.fvz.copy()
    big = (np.abs(sc.fvi[..., 0]).max(-1) > 1.0)
    z[big] = -9.0                                # behind everything else
    return sc._replace(fvz=z)


def scene_bitmask(H, W, B):
    boxlen = 0.004
    faces = [[] for _ in range(B)]
    ins = lambda r, b: faces[b].extend(quad(*r, H, W, boxlen))
    # enlarged rectangles ending on tile column 31 / 32 and starting on a 32-tile word boundary +- 1
    for i, x_hi in enumerate((511, 512, 513, 1024, 1025)):
        if x_hi <= W:
            ins((x_hi - 40, x_hi, 6 + 12 * i, 14 + 12 * i), 0)
    for i, x_lo in enumerate((495, 511, 512, 513, 1023, 1024)):
        if x_lo + 40 <= W:
            ins((x_lo, x_lo + 40, 70 - 10 * i, 78 - 10 * i), B - 1)
    if H >= 1040:
        # (tile rows x words): 64 x 1 and 32 x 2 in both views; 65 x 1 and 33 x 2 in view 0 only
        for b in range(B):
            ins((40, 200, 0, 1024), b)
            ins((500, 530, 512, 1024), b)
        ins((1100, 1200, 0, 1025), 0)
        ins((1000, 1040, 0, 528), 0)
    return finish(faces, H, W, boxlen=boxlen, seed=W + B)


def scene_culled():
    fvz, fvi, fnz = synthetic.icosphere_views(2, 3, seed=35)
    rng = np.random.default_rng(36)
    fnz = fnz.copy()
    fnz[0, rng.uniform(size=fnz.shape[1]) < 0.4] = -1.0      # front faces culled too
    fnz[1] = -np.abs(fnz[1]) - 1.0                            # a view with every face culled
    return Case(fvz, fvi, fnz.astype(np.float32), 80, 96, 1000., 0.02)


def scene_mult(m):
    fvz, fvi, fnz = synthetic.icosphere_views(1, 3, seed=37, radius=2.6)
    return Case(fvz, fvi, fnz, 56, 72, m, 0.03)


LEVEL_SHAPES = [(16, 16), (17, 9), (64, 65), (65, 64), (256, 257), (1024, 1025), (1025, 3), (4096, 4097), (4097, 5)]
SCENES = {
    **{f"levels_{H}x{W}": functools.partial(scene_levels, H, W) for H, W in LEVEL_SHAPES},
    "promote": scene_promote,
    "max_dim_16384x16": functools.partial(scene_levels, 16384, 16),
    "max_dim_16x16384": functools.partial(scene_levels, 16, 16384),
    "max_dim_soup": scene_soup_wide,
    "mixed_warp": scene_mixed_warp,
    **{f"bitmask_{W}": functools.partial(scene_bitmask, 100, W, 1) for W in (511, 512, 513)},
    "bitmask_1536": functools.partial(scene_bitmask, 1040, 1536, 2),
    "culled": scene_culled,
    **{f"mult_{m:g}": functools.partial(scene_mult, m) for m in (0.1, 333.3, 1000.)},
}


@functools.lru_cache(maxsize=None)
def scene(name):
    return SCENES[name]()


def pixels(sc):
    return sc.fnz.shape[0] * sc.H * sc.W


# ---------------------------------------------------------------------------------------------------
def _near_boundary(lo_hi, lvl, has, L):
    """{(level, side, d)}: the rectangle's lo / hi edge lies d in {-1, 0, 1} px from a bin boundary
    of its own level (not the image's edge)."""
    found = set()
    lo, hi = lo_hi
    for l in range(L - 1):
        S = TILE << 2 * l
        sel = has & (lvl == l)
        for side, e in (("lo", lo[sel]), ("hi", hi[sel])):
            for d in (-1, 0, 1):
                k = e - d
                if ((k % S == 0) & (k > 0)).any():
                    found.add((l, side, d))
    return found


@pytest.mark.parametrize("name", list(SCENES))
def test_scene_reaches_its_branch(name):
    """Each scene reaches what the module docstring says, by the host restatement of the binning."""
    sc = scene(name)
    B, F = sc.fnz.shape
    a = analyse(sc)
    L = a["L"]
    assert L == levels_for(sc.H, sc.W) <= 6
    assert all(len(w) == 0 for w in a["fallback"])       # see the module docstring
    (h0, l0, *_), (h1, l1, *_) = a["spans"]
    print(f"\n[{name}] {B}x{sc.H}x{sc.W} F={F} L={L} kernel={'aggregating' if a['agg'] else 'plain'} "
          f"tight per level {a['levels'][0].tolist()} enlarged per level {a['levels'][1].tolist()} "
          f"view_flag {a['flag'].astype(int).tolist()}")
    if name.startswith("levels"):
        sizes = {max(shape) for shape in LEVEL_SHAPES}
        assert all((TILE << 2 * l) + 1 in sizes for l in range(5)) and TILE in sizes
    if name.startswith(("levels", "max_dim_16")):
        want = set()
        for l in range(L - 1):
            S = TILE << 2 * l
            w = 8 if l == 0 else S // 2 + 1
            want |= {(l, "hi", d) for d in (-1, 0, 1)}
            if S + 1 + w <= max(sc.H, sc.W):
                want |= {(l, "lo", d) for d in (-1, 0, 1)}
        for has, lvl, r in ((h0, l0, a["tight"]), (h1, l1, a["large"])):
            got = _near_boundary((r[0], r[1]), lvl, has, L) | _near_boundary((r[2], r[3]), lvl, has, L)
            assert want <= got, sorted(want - got)
        assert not a["agg"]
    if name == "promote":
        x0, x1, y0, y1 = (v[0, 0::2] for v in a["tight"])
        rects = promote_rects(sc.H, sc.W)
        got = l0[0, 0::2]
        assert [(int(x0[i]), int(x1[i]), int(y0[i]), int(y1[i])) for i in range(len(rects))] == [r[:4] for r in rects]
        assert got.tolist() == [r[5] for r in rects]
        kinds = {(r[4], r[5] - (r[4] in ("3x", "3y"))) for r in rects}
        for l in range(L - 1):
            assert {("2x2", l), ("1x1", l), ("3x", l), ("3y", l)} <= kinds, l
    if name.startswith("max_dim"):
        assert L == 6 and max(tiles(sc.H, sc.W)) == 1024
        if sc.W == 16384:
            assert -(-tiles(sc.H, sc.W)[0] // 32) == 32
        if name == "max_dim_soup":
            assert (a["levels"][0] > 0).all() and a["flag"].all()
            assert ((a["cells"] > 0) & (a["cells"] <= 64)).any()
    if name == "mixed_warp":
        assert a["agg"]
        lvl = l0.reshape(B, -1, 32)
        big = lvl >= 1                             # the image-sized faces; every other face is at level 0
        assert ((sc.fvi[..., 0].max(-1) > 1) == big.reshape(B, F)).all()
        for lane in (0, 15, 31):
            assert (big[0, :, lane] & (big[0].sum(1) == 1)).any(), lane
        has, _, bx0, bx1, by0, by1 = (v[0].reshape(-1, 32) for v in a["spans"][0])
        bins = [{(x0, y0) for h, x0, x1, y0, y1 in zip(*w) if h and x0 == x1 and y0 == y1}
                if (w[1] == w[2])[w[0]].all() and (w[3] == w[4])[w[0]].all() else set()
                for w in zip(has, bx0, bx1, by0, by1)]
        one_bin = np.array([len(b) == 1 for b in bins]) & ~big[0].any(1)
        assert one_bin.sum() >= 20
        hot = np.nonzero(one_bin & np.array([b == {(2, 2)} for b in bins]))[0]
        assert len(hot) >= 16 and len(set(hot // 16)) >= 3      # in three 512-thread CTAs
    if name.startswith("bitmask"):
        x_lo, x_hi = a["large"][0], a["large"][1]
        live = x_hi > x_lo
        tx0, tx1 = set((x_lo[live] >> 4).tolist()), set(((x_hi[live] - 1) >> 4).tolist())
        if sc.W >= 513:
            assert {31, 32} <= tx1
        if sc.W == 1536:
            assert {31, 32, 64} <= tx0 and {63, 64} <= tx1
            assert a["flag"].tolist() == [True, False]
            c = a["cells"]
            assert {64, 65, 66} <= set(c[0].tolist()) and (c[1] == 64).sum() == 4 and c[1].max() == 64
        else:
            assert not a["flag"].any()
    if name == "culled":
        culled = sc.fnz < 0
        assert culled[1].all() and culled[0].any() and not culled[0].all()
        assert (culled & ~h0 & h1).sum() == (culled & h1).sum() > 100
        x0, x1, y0, y1 = a["tight"]
        assert (culled & (x1 > x0) & (y1 > y0)).sum() > 100              # the tight set skips these
    if name.startswith("mult"):
        mf = np.float32(sc.m)
        for n in (sc.H, sc.W):
            assert float(mf / np.float32(n)) * n != float(mf)            # multiplier / n is rounded


# ---------------------------------------------------------------------------------------------------
def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def N(t):
    return t.detach().cpu().numpy()


@functools.lru_cache(maxsize=None)
def inputs(name, dtype="fp32", D=3):
    sc = scene(name)
    B, F = sc.fnz.shape
    ff = synthetic.random_features(B, F, D, seed=40 + D)
    rng = np.random.default_rng(41)
    g_feat = rng.uniform(-1, 1, size=(B, sc.H, sc.W, D)).astype(np.float32)
    g_soft = rng.uniform(-1, 1, size=(B, sc.H, sc.W)).astype(np.float32)
    if dtype == "bf16":
        return T(ff).to(torch.bfloat16), T(g_feat).to(torch.bfloat16), T(g_soft)
    return T(ff), T(g_feat), T(g_soft)


REF_NAMES = {("fp32", 3, 30): ("face_idx", "features", "soft_mask", "grad_fvi", "grad_ff"),
             ("fp32", 3, 100): ("soft_mask", "grad_fvi"),
             ("fp32", 1, 30): ("features",),
             ("bf16", 1, 30): ("features_bf16", "grad_ff"),
             ("bf16", 3, 30): ("features_bf16", "grad_ff")}
REF_MIN_PIXELS = 1024    # the reference's rasterize backward launches no CTA below this: no stored gradients


def ref_has_grads(sc):
    return pixels(sc) >= REF_MIN_PIXELS


def reference(name, dtype="fp32", D=3, knum=30):
    """The reference's stored outputs for one run of the scene; its live run takes the bf16 features
    (and output gradients) converted to float32, as the bf16 path computes in float32."""
    sc = scene(name)
    ff, g_feat, g_soft = inputs(name, dtype, D)
    grads = ref_has_grads(sc)

    def live():
        out = ref_cuda.dibr_forward_backward(sc.H, sc.W, T(sc.fvz), T(sc.fvi), ff.float(), T(sc.fnz),
                                             g_feat.float() if grads else None, g_soft, SIGMAINV, sc.boxlen,
                                             knum, sc.m, EPS)
        return dict(out, features_bf16=out["features"].to(torch.bfloat16))

    names = [k for k in REF_NAMES[(dtype, D, knum)] if grads or not k.startswith("grad")]
    suffix = "" if (dtype, D, knum) == ("fp32", 3, 30) else f"_{dtype}_D{D}_k{knum}"
    return ref_golden.reference(f"binm_{name}{suffix}", live, names=names, path=STORE, sample_rows=64,
                                digest_only=DIGEST_ONLY)


def traced(fn):
    _lib.trace_begin()
    try:
        out = fn()
    finally:
        ran = [k for k, _ in _lib.trace_end()]
    return out, ran


def forward_kernels(sc, sets, knum):
    """The kernels the launcher picks for a forward of the scene: binning, then the rasterizer
    (dibr_fwd2_kernel when a 32x32 tile has <= 40 faces on average and there are >= 2048 such tiles),
    then the soft mask (the fused kernel with the hit cache for knum <= kSoftFwdK)."""
    B, F = sc.fnz.shape
    ks = ["bin_faces_kernel<count>", "scan_bins_kernel", "bin_faces_kernel<fill>"]
    t32 = -(-sc.W // 32) * -(-sc.H // 32)
    ks.append("dibr_fwd2_kernel<S=2>" if sets & 1 and F <= 40 * t32 and t32 * B >= 2048 else "dibr_tile_fwd_kernel")
    if sets & 2:
        ks += ["soft_fwd_kernel", "soft_tiles_fwd_kernel<leftovers>"] if knum <= SOFT_FWD_K else ["soft_tiles_fwd_kernel"]
    return ks


def run_fused(name, dtype="fp32", D=3, knum=30, grad=False):
    """dibr_rasterization, and its backward through autograd -> (feat, soft, idx, grad_fvi, grad_ff,
    kernels of the forward)."""
    from kaolin_b200.render.mesh import dibr_rasterization
    sc = scene(name)
    ff, g_feat, g_soft = inputs(name, dtype, D)
    fvi = T(sc.fvi).requires_grad_(grad)
    ff = ff.clone().requires_grad_(grad)
    (feat, soft, idx), fwd = traced(lambda: dibr_rasterization(
        sc.H, sc.W, T(sc.fvz), fvi, ff, T(sc.fnz), SIGMAINV, sc.boxlen, knum, sc.m, EPS))
    if grad:
        torch.autograd.backward([feat, soft], [g_feat, g_soft])
        return feat, soft, idx, fvi.grad, ff.grad, fwd
    return feat, soft, idx, None, None, fwd


def backward_ran(name, knum):
    """The kernels of the backward dibr_rasterization's node runs (autograd runs it on a thread of its
    own, outside the caller's trace): the same forward and backward calls, made here."""
    from kaolin_b200.render.mesh import _host
    sc = scene(name)
    ff, g_feat, g_soft = inputs(name)
    fvi = T(sc.fvi)
    feat, idx, _, soft, ws = _host.forward(_lib.RASTER | _lib.SOFT_MASK, sc.H, sc.W, T(sc.fvz), fvi, ff, T(sc.fnz),
                                           None, sc.m, EPS, SIGMAINV, sc.boxlen * sc.m, knum)
    _, ran = traced(lambda: _host.backward(sc.H, sc.W, g_feat, g_soft, idx, None, soft, fvi, ff, sc.m, EPS,
                                           SIGMAINV, sc.boxlen * sc.m, knum, ws, True))
    return ran


def cases(knums=KNUMS):
    return [(n, k) for n in SCENES for k in knums if k == 30 or pixels(scene(n)) <= ORACLE_MAX_PIXELS]


def ids(cs):
    return [f"{n}-k{k}" for n, k in cs]


@pytest.mark.gpu
@pytest.mark.parametrize("name,knum", cases(), ids=ids(cases()))
def test_fused_forward_is_the_reference(name, knum):
    sc = scene(name)
    r = reference(name, knum=knum)
    r30 = reference(name)
    feat, soft, idx, _, _, ran = run_fused(name, knum=knum)
    assert ran == forward_kernels(sc, 3, knum), ran
    bad = [k for k, t in (("face_idx", idx), ("features", feat)) if not r30.equal(k, t)]
    bad += [] if r.equal("soft_mask", soft) else ["soft_mask"]
    assert not bad, bad
    assert (idx >= 0).any()
    feat2, soft2, idx2, *_ = run_fused(name, knum=knum)
    assert torch.equal(idx2, idx) and torch.equal(feat2.view(torch.int32), feat.view(torch.int32)) \
        and torch.equal(soft2.view(torch.int32), soft.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SCENES))
def test_rasterize_and_soft_mask_alone_are_the_reference(name):
    """rasterize (only the tight set binned) and dibr_soft_mask (only the enlarged set)."""
    from kaolin_b200.render.mesh import dibr_soft_mask, rasterize
    sc = scene(name)
    r = reference(name)
    ff, _, _ = inputs(name)
    (feat, idx), ran = traced(lambda: rasterize(sc.H, sc.W, T(sc.fvz), T(sc.fvi), ff, T(sc.fnz) >= 0, sc.m, EPS))
    assert ran == forward_kernels(sc, 1, 0), ran
    assert r.equal("face_idx", idx) and r.equal("features", feat)
    soft, ran = traced(lambda: dibr_soft_mask(T(sc.fvi), idx, SIGMAINV, sc.boxlen, 30, sc.m))
    assert ran == forward_kernels(sc, 2, 30), ran
    assert r.equal("soft_mask", soft)


FEATURE_CASES = [(n, dt, D) for n in SCENES for dt, D in (("fp32", 1), ("bf16", 1), ("bf16", 3))]


@pytest.mark.gpu
@pytest.mark.parametrize("name,dtype,D", FEATURE_CASES, ids=[f"{n}-{t}-D{D}" for n, t, D in FEATURE_CASES])
def test_feature_types(name, dtype, D):
    """D = 1 in float32, and bf16 feature storage: features as the reference's float32 result rounded
    once to bf16, grad_ff within 2^-8 of the reference's."""
    sc = scene(name)
    r, r30 = reference(name, dtype, D), reference(name)
    bf16 = dtype == "bf16"
    feat, soft, idx, g_fvi, g_ff, ran = run_fused(name, dtype, D, grad=bf16)
    assert feat.dtype == (torch.bfloat16 if bf16 else torch.float32)
    assert ran == forward_kernels(sc, 3, 30), ran
    assert r30.equal("face_idx", idx) and r30.equal("soft_mask", soft)
    assert r.equal("features_bf16" if bf16 else "features", feat)
    if bf16:
        assert g_ff.dtype == torch.bfloat16
    if bf16 and ref_has_grads(sc):
        a, b = r.pair("grad_ff", g_ff.float())
        assert float(np.abs(a - b).max()) <= BF16_TOL * max(r.scale("grad_ff"), 1e-30)


def backward_kernels(sc, D):
    """The backward of dibr_rasterization with the forward's workspace: the row walk for D <= 4 and
    W a multiple of 4 px, then the soft mask from the hit cache and the tiles it could not hold."""
    raster = ["raster_bwd_rows_kernel", "raster_bwd_finalize_kernel"] if D <= ROW_WALK_MAX_D and sc.W % RW_SLAB == 0 \
        else ["raster_bwd_kernel"]
    return raster + ["soft_bwd_runs_kernel", "dibr_tile_soft_bwd_kernel<leftovers>"]


@functools.lru_cache(maxsize=None)
def oracle_grads(name, knum):
    sc = scene(name)
    ff, g_feat, g_soft = (N(t) for t in inputs(name))
    _, _, idx, w = oracle.dibr_rasterization(sc.H, sc.W, sc.fvz, sc.fvi, ff, sc.fnz, SIGMAINV, sc.boxlen, knum,
                                             sc.m, EPS, return_weights=True)
    g_fvi, g_ff, _, _ = oracle.dibr_rasterization_backward(g_feat, g_soft, idx, w, sc.fvi, ff, SIGMAINV,
                                                           sc.boxlen, knum, sc.m, EPS)
    return g_fvi, g_ff.astype(np.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("name,knum", cases(), ids=ids(cases()))
def test_backward(name, knum):
    sc = scene(name)
    r, r30 = reference(name, knum=knum), reference(name)
    _, _, _, g_fvi, g_ff, _ = run_fused(name, knum=knum, grad=True)
    ran = backward_ran(name, knum)
    assert ran == backward_kernels(sc, 3), ran
    ours = {"grad_fvi": N(g_fvi).astype(np.float64), "grad_ff": N(g_ff).astype(np.float64)}
    refs = {"grad_fvi": r, "grad_ff": r30}
    msg = f"\n[binning {name} k{knum}]"
    if pixels(sc) <= ORACLE_MAX_PIXELS:
        orc = dict(zip(("grad_fvi", "grad_ff"), oracle_grads(name, knum)))
        for k in ("grad_fvi", "grad_ff"):
            scale = max(float(np.abs(orc[k]).max()), 1e-30)
            e = float(np.abs(ours[k] - orc[k]).max()) / scale
            msg += f" {k} vs oracle {e:.2e}"
            assert e <= GRAD_TOL, (k, e)
            if not ref_has_grads(sc):
                continue
            # on the reference's stored rows where it agrees with the oracle
            rows = refs[k].rows(k)
            a, b = refs[k].pair(k, ours[k])
            o = orc[k].reshape(orc[k].shape[0] * orc[k].shape[1], -1)[rows]
            agree = (np.abs(b - o) <= REF_AGREES * scale).all(1)
            assert agree.mean() > 0.9, (k, agree.mean())
            e_ref = float(np.abs(a - b)[agree].max()) / scale if agree.any() else 0.0
            msg += f" vs reference {e_ref:.2e}"
            assert e_ref <= GRAD_TOL, (k, e_ref)
    else:
        for k in ("grad_fvi", "grad_ff"):
            a, b = refs[k].pair(k, ours[k])
            e = float(np.abs(a - b).max()) / max(refs[k].scale(k), 1e-30)
            msg += f" {k} vs reference {e:.2e}"
            assert e <= GRAD_TOL, (k, e)
    assert np.abs(ours["grad_fvi"]).max() > 0
    print(msg)
