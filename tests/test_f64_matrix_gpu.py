"""The float64 path (dibr_b200_forward_f64 / dibr_b200_backward_f64) against the reference's own
<double> kernels, bit for bit, on scenes built to break its conservative binning.

f64_prep_kernel rounds the double bboxes of the multiplied vertices outwards to float (mins down,
maxes up, tight and enlarged) and the fp32 binning enumerates that superset of candidates;
dibr_f64_kernel then decides every candidate with the reference's double comparisons, and the soft
mask visits its candidates in face-index order through the shared soft_window / soft_sort windows,
stopping at knum.  The scenes (plain numpy, each with a host-side check that it reaches what it was
built for) are:

  ulp          double bboxes whose xmin / xmax / ymin / ymax, tight and enlarged, equal a float pixel
               centre or lie one double ulp either side of it: the half-open test includes, excludes,
               includes, and rounding those boxes to the nearest float would lose pixels.
  lattice      vertices exactly on pixel centres (edges through centres, w == 0 exactly), quads split
               into two faces in both windings, coplanar duplicates and nested coplanar faces at equal
               depth (ties go to the lowest index), faces at z = +inf, zero-area faces (collinear and
               three equal vertices), faces with |norm| near eps, at eps 1e-8 and 1e-3.
  huge         scaled vertices beyond FLT_MAX (float boxes of +-inf, clamped by bbox_to_rect, the
               double test still deciding) and scaled coordinates that are subnormal or zero in float.
  windowed     sub-pixel clusters with more than 1024 enlarged-box candidates per 16x16 tile, one
               whose first density-guessed index window is empty, at knum 1, 30 and 100.
  wide         a large boxlen: enlarged rectangles as large as the image, binned above the finest level.
  views        B = 4 with an all-culled view (fnz < 0) and a view with no valid face in the middle;
               culled faces still count in the soft mask, as the reference's soft mask ignores validity.
  mult         multipliers 1, 100, 1000, 333.3 and 0.1.  The vertices are scaled by the double
               multiplier (as the reference does in torch); the kernels get its float rounding.

Bars: face_idx, weights, features and the forward soft mask are digest-equal to the reference's on
every case.  The backward is run with each branch alone (the soft branch with and without
DIBR_B200_BINS_VALID), compared on the stored rows with the reference's rasterize and soft-mask
gradients: grad_ff and grad_fvi within 1e-13 of the gradient's scale; they are double atomics in
another order.  Both branches in one call give the sum of the two branches alone to 4e-15 of scale
(measured: at most 9.5e-16; one more rounding than two orders of the same sums).  Measured on an H100 80GB HBM3 (700 W
power limit): at most 2.0e-15 for grad_ff and 1.6e-15 for grad_fvi, so these bars are tightened from
the 1e-12 / 1e-9 of test_f64_gpu.py.  The two BINS_VALID settings compute the same sums and agree to
1e-15 of scale (measured: at most 7.2e-16).  Cases that differ from another in knum alone share its
stored rasterize outputs.

The bbox test is half-open, and a pixel centre is a float: a double xmax equal to it rounds up to
itself, so the binning already drops that pixel and `x0 >= xmax` in the double test cannot be told from
`x0 > xmax` by any input.

NaN vertices make a face absent (f64_prep_kernel and the binning drop it), where the reference's result
depends on the order it visits faces in; test_nan_vertices_gpu.py holds the float64 path to the scene
without such faces.
"""
import collections
import functools

import numpy as np
import pytest
import torch

from kaolin_b200 import _lib, synthetic
from oracle import ref_cuda, ref_golden

DEV = "cuda"
SIGMAINV = 7000.
TILE = 16
SOFT_CAP = 1024
FWD, BWD = "dibr_f64_kernel<forward>", "dibr_f64_kernel<backward>"
GFF_BAR, GXY_BAR, SAME_BAR, SUM_BAR = 1e-13, 1e-13, 1e-15, 4e-15

Case = collections.namedtuple("Case", "fvz fvi fnz ff valid H W m boxlen knum eps")


# ---------------------------------------------------------------------------------------------------
# the reference's arithmetic restated on the host
def centres(H, W, m):
    """Pixel centres as the kernels compute them, in float: x ascending, y descending."""
    mf = np.float32(m)
    px = (mf / np.float32(W)) * np.arange(1 - W, W, 2).astype(np.float32)
    py = (mf / np.float32(H)) * np.arange(H - 1, -H, -2).astype(np.float32)
    return px.astype(np.float64), py.astype(np.float64)


def boxes(fvi, m, margin):
    """(xmin, ymin, xmax, ymax) of face_vertices_image * m in double, enlarged by margin."""
    v = np.asarray(fvi, np.float64) * m
    return (v[..., 0].min(-1) - margin, v[..., 1].min(-1) - margin,
            v[..., 0].max(-1) + margin, v[..., 1].max(-1) + margin)


def rd(x):
    with np.errstate(over="ignore"):
        f = np.asarray(x, np.float64).astype(np.float32)
    return np.where(f.astype(np.float64) > x, np.nextafter(f, np.float32(-np.inf)), f)


def ru(x):
    with np.errstate(over="ignore"):
        f = np.asarray(x, np.float64).astype(np.float32)
    return np.where(f.astype(np.float64) < x, np.nextafter(f, np.float32(np.inf)), f)


def nearest(x):
    with np.errstate(over="ignore"):
        return np.asarray(x, np.float64).astype(np.float32)


def rects(H, W, m, xmin, ymin, xmax, ymax):
    """Pixel rectangles [x_lo, x_hi) x [y_lo, y_hi) passing the half-open test
    !(x0 < xmin || x0 >= xmax || y0 < ymin || y0 >= ymax), compared in double (float boxes widen exactly)."""
    px, py = centres(H, W, m)
    rising = py[::-1]
    f = lambda a: np.asarray(a, np.float64)
    return (np.searchsorted(px, f(xmin), "left"), np.searchsorted(px, f(xmax), "left"),
            H - np.searchsorted(rising, f(ymax), "left"), H - np.searchsorted(rising, f(ymin), "left"))


def pixel_sets(sc, margin):
    """-> (double, conservative float, nearest float) pixel rectangles of every face's box."""
    b = boxes(sc.fvi, sc.m, margin)
    return (rects(sc.H, sc.W, sc.m, *b),
            rects(sc.H, sc.W, sc.m, rd(b[0]), rd(b[1]), ru(b[2]), ru(b[3])),
            rects(sc.H, sc.W, sc.m, *(nearest(a) for a in b)))


def contains(outer, inner):
    """Every pixel of each inner rectangle lies in the outer one (empty inner rectangles always)."""
    ox0, ox1, oy0, oy1 = outer
    ix0, ix1, iy0, iy1 = inner
    empty = (ix1 <= ix0) | (iy1 <= iy0)
    return empty | ((ox0 <= ix0) & (ix1 <= ox1) & (oy0 <= iy0) & (iy1 <= oy1))


def preimage(t, m, margin=0.0):
    """An unscaled coordinate u with fl(fl(u * m) + margin) == t, or None."""
    for u in ((t - margin) / m, t / m - margin / m):
        up = dn = u
        for _ in range(64):
            for c in (up, dn):
                if (c * m) + margin == t:
                    return c
            up, dn = np.nextafter(up, np.inf), np.nextafter(dn, -np.inf)
    return None


# ---------------------------------------------------------------------------------------------------
# scenes
def features(B, F, seed, D=2):
    return np.random.default_rng(seed).uniform(-1, 1, size=(B, F, 3, D))


def finish(parts, H, W, m, boxlen=0.02, knum=30, eps=1e-8, seed=0, valid=None):
    """parts: per view, a list of (fvz (n,3), fvi (n,3,2), fnz (n,)) -> Case with double arrays."""
    st = [tuple(np.concatenate([np.asarray(p[i], np.float64) for p in view]) for i in range(3)) for view in parts]
    fvz, fvi, fnz = (np.stack([v[i] for v in st]) for i in range(3))
    return Case(fvz, fvi, fnz, features(*fvz.shape[:2], seed), valid, H, W, m, boxlen, knum, eps)


ULP_KINDS = [(axis, side, delta, large) for large in (False, True) for axis in (0, 1)
             for side in ("min", "max") for delta in (0, 1, -1)]


def _ulp_face(t_along, c_cross, axis, side, pitch, m, margin):
    """A face whose extreme coordinate along `axis` on `side` scales to t_along (after +-margin), with
    that vertex at the cross coordinate c_cross; None if t_along has no preimage."""
    sgn = 1.0 if side == "max" else -1.0
    u = preimage(t_along, m, sgn * margin)
    uc = preimage(c_cross, m)
    if u is None or uc is None:
        return None
    depth = (0.3 * pitch if margin else 1.5 * pitch) / m       # enlarged faces stay between pixel columns
    back = u - sgn * depth
    spread = 1.5 * pitch / m
    pts = [(u, uc), (back, uc - spread), (back, uc + spread)]
    if axis == 1:
        pts = [(b, a) for a, b in pts]
    return np.array(pts)


def scene_ulp():
    H = W = 40
    m = 1000.
    boxlen = 0.008            # margin 8 in scaled units: a third of the pixel pitch of 50
    margin = boxlen * m
    px, py = centres(H, W, m)
    pitch = px[1] - px[0]
    spots = [(ix, iy) for iy in range(2, H - 2, 5) for ix in range(2, W - 2, 5)]
    rng = np.random.default_rng(10)
    faces, used, targets = [], 0, []
    for kind in ULP_KINDS:
        axis, side, delta, large = kind
        while True:
            ix, iy = spots[used]
            used += 1
            x0, y0 = px[ix], py[iy]
            along, cross = (x0, y0) if axis == 0 else (y0, x0)
            t = along if delta == 0 else np.nextafter(along, np.inf * delta)
            f = _ulp_face(t, cross, axis, side, pitch, m, margin if large else 0.0)
            if f is not None:
                break
        faces.append(f)
        targets.append((ix, iy))
    n = len(faces)
    fvz = rng.uniform(-3, -1, size=(n, 3))
    sc = finish([[(fvz, np.stack(faces), np.ones(n))]], H, W, m, boxlen=boxlen, knum=40, seed=11)
    return sc._replace(valid=None), targets


def scene_lattice(eps):
    H = W = 64
    m = 1.0
    px, py = centres(H, W, m)
    P = lambda i, j: (px[i], py[j])
    parts = []
    z = lambda n, v: np.full((n, 3), v)
    # quads split along a diagonal through pixel centres, CCW in the top half, CW below; coplanar
    quad = lambda i, j, s: [[P(i, j), P(i + s, j), P(i + s, j + s)], [P(i, j), P(i + s, j + s), P(i, j + s)]]
    # (z = 0 interpolates to exactly 0 whatever the weights: equal depths are exact ties)
    q1 = quad(2, 2, 6)
    q2 = [f[::-1] for f in quad(2, 18, 6)]
    parts.append((z(4, 0.0), np.array(q1 + q2), np.ones(4)))
    # coplanar duplicates, and a small face inside a big one at the same depth, the big one first: it
    # spans more than 2x2 of the finest bins, so it is binned one level up and visited after the small one
    dup = [[P(12, 2), P(18, 2), P(12, 8)]] * 2
    nest_big = [[P(4, 34), P(60, 34), P(4, 62)]]
    nest_small = [[P(8, 38), P(14, 38), P(8, 44)]]
    parts.append((z(4, 0.0), np.array(dup + nest_big + nest_small), np.ones(4)))
    # faces at z = +inf, vertices off the lattice so that no centre lies on an edge (w > 0 inside)
    h = (px[1] - px[0]) / 2
    inf = [[(px[12] + h * 0.3, py[12] + h * 0.7), (px[20] + h * 0.6, py[13] + h * 0.1), (px[13] + h * 0.2, py[20] + h * 0.9)]] * 2
    parts.append((z(2, np.inf), np.array(inf), np.ones(2)))
    # zero-area: collinear through centres, and three equal vertices on a centre
    col = [[P(3, 28), P(6, 28), P(10, 28)], [P(3, 25), P(5, 27), P(7, 29)]]
    pt = [[P(14, 26)] * 3]
    parts.append((z(3, 0.5), np.array(col + pt), np.ones(3)))
    # tiny faces around a centre, |norm| ~ 1e-8 and ~ 1e-3 (scaled units)
    tiny = []
    for s in (1e-4, 3e-2):
        for (i, j) in ((24, 20), (27, 24)):
            x, y = P(i, j)
            tiny.append([(x - s, y - s), (x + s, y - s * 0.5), (x - s * 0.3, y + s)])
    parts.append((z(4, -0.5), np.array(tiny), np.ones(4)))
    return finish([parts], H, W, m, boxlen=0.05, knum=50, eps=eps, seed=12)


def scene_huge():
    H = W = 33                       # odd: the middle pixel centre is exactly 0
    m = 1000.
    B = 1e36
    faces = [[(-B, -B), (0.2, -B), (0.2, B)],                    # beyond FLT_MAX once scaled: +-inf float boxes
             [(-B, -B), (-B, B), (-0.3, 0.1)],                   # a wedge from far left, its tip on screen
             [(2 * B, 0.0), (3 * B, 0.0), (2 * B, B)],           # all of it beyond FLT_MAX: nothing
             [(-1e-49, -1e-49), (1e-49, -1e-49), (0.0, 1e-49)],  # 1e-46 scaled: below the float subnormals
             [(-1e-43, -1e-43), (1e-43, -1e-43), (0.0, 1e-43)]]  # 1e-40 scaled: subnormal in float
    fvz = np.array([[-5.0] * 3, [-4.0] * 3, [-1.0] * 3, [-0.5] * 3, [-0.6] * 3])
    return finish([[(fvz, np.array(faces), np.ones(5))]], H, W, m, boxlen=0.2, knum=10, seed=13)


def _cluster(n, centre, rng):
    c = np.asarray(centre) + rng.uniform(-0.1, 0.1, size=(n, 1, 2))
    return rng.uniform(-3, -1, size=(n, 3)), c + rng.normal(scale=0.004, size=(n, 3, 2)), np.ones(n)


def scene_windowed(knum):
    rng = np.random.default_rng(14)
    z, xy, n = synthetic.triangle_soup(1, 2000, seed=74, coverage=1.0)
    left = (z[0], xy[0].astype(np.float64) * 0.4 - 0.5 + rng.uniform(-1e-9, 1e-9, xy[0].shape), n[0])
    return finish([[left, _cluster(1100, (0.75, -0.75), rng), _cluster(1100, (0.75, 0.75), rng)]],
                  64, 64, 1000., boxlen=0.02, knum=knum, seed=15)


def _mesh(views, level, seed, radius=3.0):
    fvz, fvi, fnz = synthetic.icosphere_views(views, level, seed=seed, radius=radius)
    rng = np.random.default_rng(seed + 1)
    j = lambda a: a.astype(np.float64) + rng.uniform(-1e-9, 1e-9, a.shape)
    return j(fvz), j(fvi), fnz.astype(np.float64)


def scene_wide():
    fvz, fvi, fnz = _mesh(2, 2, 16)
    return finish([[(fvz[b], fvi[b], fnz[b])] for b in range(2)], 96, 80, 1000., boxlen=1.0, knum=30, seed=17)


def scene_views():
    fvz, fvi, fnz = _mesh(4, 2, 18)
    fnz[1] = -np.abs(fnz[1]) - 1.0               # every face of view 1 culled by its normal
    valid = np.ones(fnz.shape, bool)
    valid[2] = False                             # no valid face in view 2
    valid[3] = np.random.default_rng(19).uniform(size=valid.shape[1]) < 0.7
    sc = finish([[(fvz[b], fvi[b], fnz[b])] for b in range(4)], 48, 56, 1000., boxlen=0.04, knum=30, seed=20)
    return sc._replace(valid=valid)


def scene_mult(m):
    fvz, fvi, fnz = _mesh(1, 1, 21, radius=2.6)
    return finish([[(fvz[0], fvi[0], fnz[0])]], 64, 72, m, boxlen=0.03, knum=30, seed=22)


SCENES = {
    "ulp": lambda: scene_ulp()[0],
    "lattice_eps1e-8": lambda: scene_lattice(1e-8),
    "lattice_eps1e-3": lambda: scene_lattice(1e-3),
    "huge": scene_huge,
    "windowed_k1": lambda: scene_windowed(1),
    "windowed_k30": lambda: scene_windowed(30),
    "windowed_k100": lambda: scene_windowed(100),
    "wide": scene_wide,
    "views": scene_views,
    "lattice_kall": lambda: scene_lattice(1e-8)._replace(knum=5000),
    **{f"mult_{m:g}": functools.partial(scene_mult, m) for m in (1., 100., 1000., 333.3, 0.1)},
}


@functools.lru_cache(maxsize=None)
def scene(name):
    return SCENES[name]()


def raster_valid(sc):
    v = sc.fnz >= 0
    return v if sc.valid is None else v & sc.valid


def tile_candidates(sc, rect):
    """(B, tiles_y, tiles_x) number of faces whose rectangle meets each 16x16 tile."""
    x0, x1, y0, y1 = rect
    B = sc.fvi.shape[0]
    nty, ntx = -(-sc.H // TILE), -(-sc.W // TILE)
    out = np.zeros((B, nty, ntx), np.int64)
    for b in range(B):
        for f in np.nonzero((x1[b] > x0[b]) & (y1[b] > y0[b]))[0]:
            out[b, y0[b, f] // TILE:(y1[b, f] - 1) // TILE + 1, x0[b, f] // TILE:(x1[b, f] - 1) // TILE + 1] += 1
    return out


# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SCENES))
def test_scene_reaches_its_branch(name):
    """Each scene has the property the module docstring gives it; the conservative float boxes always
    hold the double ones."""
    sc = scene(name)
    B, F = sc.fvi.shape[:2]
    for margin in (0.0, sc.boxlen * sc.m):
        dbl, cons, near = pixel_sets(sc, margin)
        assert contains(cons, dbl).all()
    if name == "ulp":
        _, targets = scene_ulp()
        px, py = centres(sc.H, sc.W, sc.m)
        for large in (False, True):
            dbl, cons, near = pixel_sets(sc, sc.boxlen * sc.m if large else 0.0)
            lost = ~contains(near, dbl)[0]
            gained = ~contains(dbl, near)[0]
            for f, (kind, (ix, iy)) in enumerate(zip(ULP_KINDS, targets)):
                axis, side, delta, lg = kind
                if lg != large:
                    continue
                x0, x1, y0, y1 = (a[0, f] for a in dbl)
                inside = x0 <= ix < x1 and y0 <= iy < y1
                # half-open: the min side includes x0 == min, the max side excludes x0 == max
                assert inside == ((side == "min") != (delta == 1) if delta else side == "min"), (kind, inside)
                b = boxes(sc.fvi[:, f], sc.m, sc.boxlen * sc.m if large else 0.0)
                centre = px[ix] if axis == 0 else py[iy]
                along = b[(0 if side == "min" else 2) + axis][0]
                assert along == (centre if delta == 0 else np.nextafter(centre, np.inf * delta)), kind
            assert lost.sum() >= 2 and gained.sum() >= 2, (large, lost.sum(), gained.sum())
    if name.startswith("lattice"):
        px, py = centres(sc.H, sc.W, sc.m)
        v = sc.fvi[0] * sc.m
        on = np.isin(v[..., 0], px) & np.isin(v[..., 1], py)
        assert on[:8].all() and on[8:].sum() >= 9
        assert np.isinf(sc.fvz[0]).any()
        x0, x1, y0, y1 = (a[0, 6:8] for a in pixel_sets(sc, 0.0)[1])
        big = lambda a, b: ((b - 1) >> 4) - (a >> 4) > 1
        assert big(x0[0], x1[0]) and not big(x0[1], x1[1]) and not big(y0[1], y1[1])   # binned at different levels
        assert x0[0] <= x0[1] and x1[1] <= x1[0] and y0[0] <= y0[1] and y1[1] <= y1[0]
        e = (v[:, 1] - v[:, 0])
        area = e[:, 0] * (v[:, 2, 1] - v[:, 0, 1]) - e[:, 1] * (v[:, 2, 0] - v[:, 0, 0])
        assert (area == 0).sum() == 3
        assert (np.abs(area) < 1e-7).any() and ((np.abs(area) > 1e-4) & (np.abs(area) < 1e-2)).any()
    if name == "huge":
        with np.errstate(over="ignore", invalid="ignore"):
            v = sc.fvi[0] * sc.m
            assert (np.abs(v) > np.finfo(np.float32).max).any(axis=(1, 2))[:3].all()
            tiny = np.abs(v[3:][v[3:] != 0])
            assert (nearest(tiny) == 0).any() and (tiny < np.finfo(np.float32).tiny).all()
        dbl, _, near = pixel_sets(sc, 0.0)
        assert not contains(near, dbl)[0, 3]           # the nearest float box loses the middle pixel
        assert dbl[0][0, 3] <= sc.W // 2 < dbl[1][0, 3]
    if name.startswith("windowed"):
        dbl, cons, _ = pixel_sets(sc, sc.boxlen * sc.m)
        cand = tile_candidates(sc, cons)
        big = list(zip(*np.nonzero(cand[0] > SOFT_CAP)))
        assert len(big) == 2
        x0, x1, y0, y1 = (a[0] for a in cons)
        firsts = []
        for ty, tx in big:
            meets = np.nonzero((x1 > x0) & (y1 > y0) & (x0 // TILE <= tx) & (tx <= (x1 - 1) // TILE)
                               & (y0 // TILE <= ty) & (ty <= (y1 - 1) // TILE))[0]
            firsts.append(int((meets <= max(F * SOFT_CAP * 3 // (len(meets) * 4), 1) - 1).sum()))
        assert min(firsts) == 0 and max(firsts) > 0, firsts
    if name == "wide":
        _, cons, _ = pixel_sets(sc, sc.boxlen * sc.m)
        x0, x1, y0, y1 = cons
        span = lambda lo, hi: ((hi - 1) >> 4) - (lo >> 4)          # in 16-pixel bins, minus one
        assert ((span(x0, x1) > 1) & (span(y0, y1) > 1)).mean() > 0.5      # binned above the finest level
        assert ((x0 == 0) & (x1 == sc.W) & (y0 == 0) & (y1 == sc.H)).any()  # a rectangle the size of the image
    if name == "views":
        v = raster_valid(sc)
        assert not v[1].any() and not v[2].any() and v[0].any() and v[3].any() and not v[3].all()
    if name == "lattice_kall":
        assert sc.knum > F


# ---------------------------------------------------------------------------------------------------
def D(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@functools.lru_cache(maxsize=None)
def grads(name):
    sc = scene(name)
    B = sc.fvi.shape[0]
    rng = np.random.default_rng(30)
    return rng.uniform(-1, 1, size=(B, sc.H, sc.W, sc.ff.shape[-1])), rng.uniform(-1, 1, size=(B, sc.H, sc.W))


NAMES = ("face_idx", "features", "weights", "soft_mask", "grad_ff", "grad_fvi_raster", "grad_fvi_soft")
SOFT_NAMES = ("soft_mask", "grad_fvi_soft")
# cases that differ from another one in knum alone: their rasterize outputs and gradients are that case's
RASTER_FROM = {"windowed_k1": "windowed_k30", "windowed_k100": "windowed_k30", "lattice_kall": "lattice_eps1e-8"}


def raster_reference(name):
    return reference(RASTER_FROM.get(name, name))


@functools.lru_cache(maxsize=None)
def reference(name):
    sc = scene(name)
    g_feat, g_soft = grads(name)

    def live():
        valid = D(raster_valid(sc))
        fvi, ff = D(sc.fvi), D(sc.ff)
        feat, idx, w = ref_cuda.rasterize_forward(sc.H, sc.W, D(sc.fvz), fvi, ff, valid, sc.m, sc.eps)
        soft, fvi_m, prob, cidx, ctype = ref_cuda.soft_mask_forward(fvi, idx, SIGMAINV, sc.boxlen, sc.knum, sc.m)
        gxy_r, gff = ref_cuda.rasterize_backward(D(g_feat), feat, idx, w, fvi, ff, sc.eps)
        gxy_s = ref_cuda.soft_mask_backward(D(g_soft), soft, idx, prob, cidx, ctype, fvi_m, SIGMAINV, sc.m)
        return {"face_idx": idx, "features": feat, "weights": w, "soft_mask": soft,
                "grad_ff": gff, "grad_fvi_raster": gxy_r, "grad_fvi_soft": gxy_s}

    small = sc.fvi.shape[0] * sc.H * sc.W <= 4096
    return ref_golden.reference(f"f64m_{name}", live, names=SOFT_NAMES if name in RASTER_FROM else NAMES,
                                full=("face_idx",) if small else ())


def forward(name):
    """dibr_b200_forward_f64, RASTER | SOFT_MASK, as the public API calls it -> (feat, idx, w, soft, ws)."""
    from kaolin_b200.render.mesh import _host
    sc = scene(name)
    valid = None if sc.valid is None else D(sc.valid.astype(np.uint8))
    _lib.trace_begin()
    try:
        out = _host.forward(_lib.RASTER | _lib.SOFT_MASK, sc.H, sc.W, D(sc.fvz), D(sc.fvi), D(sc.ff), D(sc.fnz),
                            valid, sc.m, sc.eps, SIGMAINV, sc.boxlen * sc.m, sc.knum)
    finally:
        ran = [k for k, _ in _lib.trace_end()]
    assert FWD in ran, ran
    return out


def rel(r, name, ours):
    a, b = r.pair(name, ours)
    return float(np.abs(a - b).max()) / max(r.scale(name), 1e-300)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SCENES))
def test_forward_is_the_reference_bit_for_bit(name):
    sc = scene(name)
    feat, idx, w, soft, _ = forward(name)
    r, rr = reference(name), raster_reference(name)
    bad = [k for k, t in (("face_idx", idx), ("weights", w), ("features", feat)) if not rr.equal(k, t)]
    bad += [] if r.equal("soft_mask", soft) else ["soft_mask"]
    assert not bad, bad
    assert (idx >= 0).any() and ((soft > 0) & (soft < 1)).any()
    if name == "ulp":
        _, targets = scene_ulp()
        i = idx[0].cpu().numpy()
        for f, (kind, (ix, iy)) in enumerate(zip(ULP_KINDS, targets)):
            axis, side, delta, large = kind
            if not large:       # the pixel the bbox test decides is rasterized by exactly that face, or not
                assert (i[iy, ix] == f) == ((side == "min") != (delta == 1) if delta else side == "min"), kind
    if sc.valid is None:
        # the public API takes the same path
        from kaolin_b200.render.mesh import dibr_rasterization
        f2, s2, i2 = dibr_rasterization(sc.H, sc.W, D(sc.fvz), D(sc.fvi), D(sc.ff), D(sc.fnz), SIGMAINV,
                                        sc.boxlen, sc.knum, sc.m, sc.eps)
        assert torch.equal(i2, idx) and torch.equal(f2, feat) and torch.equal(s2, soft)


BRANCHES = ["both", "raster", "soft", "soft_fresh"]
CASES = [(n, b) for n in SCENES for b in BRANCHES if not (b == "raster" and n in RASTER_FROM)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,branch", CASES, ids=[f"{n}-{b}" for n, b in CASES])
def test_backward(name, branch):
    """Both branches, each alone, the soft branch with the forward's bins (BINS_VALID) and rebuilding them.
    Each branch alone is held to the reference; both together are the sum of the two, in one kernel."""
    from kaolin_b200.render.mesh import _host
    sc = scene(name)
    feat, idx, w, soft, ws = forward(name)
    gf, gs = (D(g) for g in grads(name))
    fresh = branch == "soft_fresh"

    def run(g_feat, g_soft, ws, valid_bins):
        _lib.trace_begin()
        try:
            out = _host.backward(sc.H, sc.W, g_feat, g_soft, idx, w, soft, D(sc.fvi), D(sc.ff), sc.m, sc.eps,
                                 SIGMAINV, sc.boxlen * sc.m, sc.knum, ws, valid_bins)
        finally:
            ran = [k for k, _ in _lib.trace_end()]
        assert BWD in ran, ran
        return out

    rr, rs = raster_reference(name), reference(name)
    msg = f"\n[f64 matrix {name} {branch}]"
    if branch == "both":
        g_fvi, g_ff = run(gf, gs, ws, True)
        g_r, _ = run(gf, None, ws, True)
        g_s, _ = run(None, gs, ws, True)
        e_r, e_s = rel(rr, "grad_fvi_raster", g_r), rel(rs, "grad_fvi_soft", g_s)
        same = float((g_fvi - (g_r + g_s)).abs().max()) / max(rr.scale("grad_fvi_raster"), rs.scale("grad_fvi_soft"), 1e-300)
        msg += f" grad_fvi_raster {e_r:.2e} grad_fvi_soft {e_s:.2e} both vs the sum {same:.2e}"
        assert e_r <= GXY_BAR and e_s <= GXY_BAR, (e_r, e_s)
        assert same <= SUM_BAR, same
    elif branch == "raster":
        g_fvi, g_ff = run(gf, None, ws, True)
        e_xy = rel(rr, "grad_fvi_raster", g_fvi)
        msg += f" grad_fvi_raster {e_xy:.2e}"
        assert e_xy <= GXY_BAR, e_xy
        assert g_fvi.any() or rr.scale("grad_fvi_raster") == 0
    else:
        g_fvi, g_ff = run(None, gs, None if fresh else ws, not fresh)
        other, _ = run(None, gs, ws if fresh else None, fresh)
        e_xy = rel(rs, "grad_fvi_soft", g_fvi)
        same = float((other - g_fvi).abs().max()) / max(rs.scale("grad_fvi_soft"), 1e-300)
        msg += f" grad_fvi_soft {e_xy:.2e} BINS_VALID vs rebuilt {same:.2e}"
        assert e_xy <= GXY_BAR, e_xy
        assert same <= SAME_BAR, same
        assert g_fvi.any() or rs.scale("grad_fvi_soft") == 0
        assert not g_ff.any()
    if not branch.startswith("soft"):
        e_ff = rel(rr, "grad_ff", g_ff)
        msg += f" grad_ff {e_ff:.2e}"
        assert e_ff <= GFF_BAR, e_ff
    print(msg)
