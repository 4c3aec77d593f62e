"""NaN vertex coordinates: a tainted face is absent, in every entry point, kernel path and storage type.

A face is tainted when any of its nine coordinates is NaN: the three of face_vertices_z or the six of
face_vertices_image.  Such a face never wins a pixel, is never a soft-mask candidate, and its rows of
grad_face_vertices_image and grad_face_features are exactly zero; every other output and gradient is
that of the same call on the scene with the tainted faces deleted, face_idx mapped back to the
original indices.  bin_faces_kernel (dibr_b200.cu) drops a tainted face from both bin sets, and
f64_prep_kernel (dibr_f64.cuh) gives a face with a NaN depth NaN float vertices so that the float64
path's binning drops it too; no per-pixel loop sees such a face.  Without that, fminf / fmaxf bin a
face with one NaN vertex on the rectangle of its finite vertices, the inside test passes its NaN
weights, and `!(z <= best)` lets its NaN depth win and hand the pixel to every later covering face.
The reference's result on such input depends on its face loop order (DESIGN.md, NaN vertices).

The stripped scene keeps the tainted faces' slots, filled with faces far off screen (they bin
nowhere), so both calls have the same shape and take the same kernels.  Scenes:

  coord_k       an icosphere view with one front face tainted in coordinate k (z0 z1 z2 x0 y0 x1 y1 x2
                y2), and in all nine.
  bins          tainted faces whose finite vertices span more than 2x2 bins, the whole image (the
                coarsest level), and end on a 64 px bin border or one pixel either side of it, over
                finite quads at the same places.
  dense         an icosphere at >= 32 faces per 16x16 tile (the aggregating bin kernel), tainted faces
                in lanes 0, 15 and 31 of several warps.
  z_front       the frontmost face over finite ones, NaN only in z: the case the reference's loop order
                decides.
  culled        tainted faces among culled ones (face_normals_z < 0) and, for rasterize, valid_faces.
  batch_view    one view of three fully tainted: it is empty, and its neighbours are bit-identical to
                rendering them without it.
  all           every face tainted.
  c4_shard      32 x 1024^2 views of a level-5 icosphere (bench.py's workload), 1 % tainted: the
                persistent dibr_fwd2_kernel, the fused soft-mask forward, the hit-cache backward.
  wide_2048     a 2048^2 view with 1 % tainted and a full-image sliver whose enlarged rectangle is too
                big for the per-tile bitmask (view_flag).

Paths: dibr_rasterization at knum 30 (fused soft-mask forward) and 100 (single kernel) with float32 and
bf16 features and in float64; rasterize alone with and without valid_faces; dibr_soft_mask alone;
backward through both outputs and through each alone; the soft-mask backward from the hit cache and
recomputed (CACHE_TILE_FRACTION = 0); the view-chunked backward; one call of
make_graphed_dibr_rasterization.

Bars: (a) this library on the stripped scene, face_idx, features and soft mask bit-equal, gradients
within 1e-5 of the gradient's scale (the atomics' order differs) and exactly zero on tainted rows;
(b) the reference's kernels on the stripped scene (tests/golden/ref_cuda_nan.npz), face_idx, features
and soft mask bit-equal, gradients within 3e-5 of scale on its stored rows; (c) the double-accumulating
C oracle on the stripped scene, gradients within 3e-5 of scale.  The deviation is recorded: on z_front
and on a face with NaN x the reference, run on the tainted scene, gives pixels to the tainted face, and
ours differ there.  Reruns are byte-identical, the call synchronises nothing with the host, and nothing
is printed on stderr.
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

pytestmark = pytest.mark.gpu

DEV = "cuda"
SIGMAINV, EPS = 7000., 1e-8
SELF_TOL, GRAD_TOL, BF16_TOL = 1e-5, 3e-5, 2.0 ** -8
ORACLE_MAX_WORK = 1 << 31          # pixels x faces the C oracle walks
STORE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_cuda_nan.npz")
OFF = 5.0                          # x of the faces that fill deleted slots: far right of the image

# nan: (B, F, 9) bool, coordinates z0 z1 z2 x0 y0 x1 y1 x2 y2
Case = collections.namedtuple("Case", "fvz fvi fnz H W m boxlen nan")


# ---------------------------------------------------------------------------------------------------
# scenes
def X(k, W):
    """x of the boundary between pixel columns k - 1 and k."""
    return (2.0 * k - W) / W


def Y(k, H):
    return (H - 2.0 * k) / H


def front_faces(fvi, fnz, n):
    """n front faces of view 0, the largest on screen first."""
    v = fvi[0]
    area = 0.5 * np.abs((v[:, 1, 0] - v[:, 0, 0]) * (v[:, 2, 1] - v[:, 0, 1])
                        - (v[:, 2, 0] - v[:, 0, 0]) * (v[:, 1, 1] - v[:, 0, 1]))
    area = np.where(fnz[0] >= 0, area, -1)
    return np.argsort(-area, kind="stable")[:n]


def case(fvz, fvi, fnz, H, W, nan, m=1000., boxlen=0.02):
    return Case(fvz.astype(np.float32), fvi.astype(np.float32), fnz.astype(np.float32), H, W, m, boxlen, nan)


def scene_coord(k):
    fvz, fvi, fnz = synthetic.icosphere_views(1, 3, seed=81)
    nan = np.zeros(fvz.shape + (3,), bool).reshape(1, -1, 9)
    f = front_faces(fvi, fnz, 1)[0]
    nan[0, f, :] = True if k == 9 else np.arange(9) == k
    return case(fvz, fvi, fnz, 96, 80, nan)


def scene_bins():
    """256 x 256 (3 levels: 16, 64 and 256 px).  Tainted faces have one NaN vertex (in x, y or z),
    the other two at opposite corners of the rectangle their fminf / fmaxf box would be."""
    H = W = 256
    faces, taint = [], []

    def seg(x0, x1, y0, y1, k):
        """NaN in coordinate k of vertex 2 (x2 = 7, y2 = 8, z2 = 2)."""
        faces.append([(X(x0, W), Y(y0, H)), (X(x1, W), Y(y1, H)), (X(x0, W), Y(y1, H))])
        taint.append(k)

    def quad(x0, x1, y0, y1):
        a, b, c, d = (X(x0, W), Y(y0, H)), (X(x1, W), Y(y0, H)), (X(x0, W), Y(y1, H)), (X(x1, W), Y(y1, H))
        faces.extend([[a, b, c], [b, d, c]])
        taint.extend([-1, -1])

    quad(20, 236, 30, 226)                          # finite faces below everything tainted
    seg(10, 100, 12, 90, 7)                         # 90 x 78 px: 3 x 3 bins of 64 px, level 2
    seg(0, W, 0, H, 8)                              # image-wide: the coarsest level
    seg(0, W, 120, 124, 2)                          # an image-wide strip
    for i, e in enumerate((63, 64, 65, 127, 128, 129)):
        k = (7, 8, 2)[i % 3]
        seg(e - 20, e, 140 + 18 * (i % 3), 150 + 18 * (i % 3), k)            # hi x edge at e
        seg(e, e + 20, 200 + 8 * (i % 3), 206 + 8 * (i % 3), k)              # lo x edge at e
        seg(40 + 10 * i, 48 + 10 * i, e - 12, e, k)                          # hi y edge at e
        seg(160 + 10 * i, 168 + 10 * i, e, e + 12, k)                        # lo y edge at e
        quad(e - 6, e + 6, 100 + 3 * i, 104 + 3 * i)                         # finite, on the border
    F = len(faces)
    fvi = np.array(faces)
    rng = np.random.default_rng(82)
    fvz = np.repeat(rng.uniform(-3, -1, (1, F, 1)), 3, 2)
    fvz[0, 0:2] = -8.0                              # the big finite quad is at the back
    nan = np.zeros((1, F, 9), bool)
    for f, k in enumerate(taint):
        if k >= 0:
            nan[0, f, k] = True
    return case(fvz, fvi[None], np.ones((1, F)), H, W, nan, boxlen=0.01)


def scene_dense():
    fvz, fvi, fnz = synthetic.icosphere_views(2, 5, seed=83)          # 20480 faces at 64 x 64: 1280 per tile
    nan = np.zeros((2, fvz.shape[1], 9), bool)
    rng = np.random.default_rng(84)
    for b in range(2):
        for w in rng.choice(fvz.shape[1] // 32, 40, replace=False):
            for lane in (0, 15, 31):
                nan[b, 32 * w + lane, rng.integers(9)] = True
    return case(fvz, fvi, fnz, 64, 64, nan)


def scene_z_front():
    """A face in front of the sphere with NaN depth at one vertex; the sphere's faces come after it."""
    fvz, fvi, fnz = synthetic.icosphere_views(1, 3, seed=85)
    F = fvz.shape[1]
    front = np.array([[[-0.98, -0.98], [0.98, -0.98], [0.0, 0.98]]], np.float32)   # beyond the silhouette
    fvi = np.concatenate([front[None], fvi], 1)
    fvz = np.concatenate([np.full((1, 1, 3), -0.5, np.float32), fvz], 1)
    fnz = np.concatenate([np.ones((1, 1), np.float32), fnz], 1)
    nan = np.zeros((1, F + 1, 9), bool)
    nan[0, 0, 1] = True
    return case(fvz, fvi, fnz, 96, 96, nan)


def scene_nan_x():
    """The same, with the NaN in x of one vertex: the reference's bbox test passes every pixel."""
    sc = scene_z_front()
    nan = np.zeros_like(sc.nan)
    nan[0, 0, 5] = True
    return sc._replace(nan=nan)


def scene_culled():
    fvz, fvi, fnz = synthetic.icosphere_views(2, 3, seed=86)
    rng = np.random.default_rng(87)
    fnz = fnz.copy()
    fnz[rng.uniform(size=fnz.shape) < 0.3] = -1.0
    nan = np.zeros((2, fvz.shape[1], 9), bool)
    pick = rng.uniform(size=fnz.shape) < 0.15
    nan[pick, rng.integers(9, size=pick.sum())] = True
    assert (pick & (fnz < 0)).any() and (pick & (fnz >= 0)).any()
    return case(fvz, fvi, fnz, 80, 96, nan)


def scene_batch_view():
    fvz, fvi, fnz = synthetic.icosphere_views(3, 3, seed=88)
    F = fvz.shape[1]
    nan = np.zeros((3, F, 9), bool)
    nan[1, np.arange(F), np.random.default_rng(89).integers(9, size=F)] = True
    return case(fvz, fvi, fnz, 72, 88, nan)


def scene_all():
    fvz, fvi, fnz = synthetic.icosphere_views(2, 3, seed=90)
    nan = np.zeros((2, fvz.shape[1], 9), bool)
    nan[..., 4] = True
    nan[1, ::2, 0] = True
    return case(fvz, fvi, fnz, 64, 80, nan)


def scattered(fvz, percent, seed):
    rng = np.random.default_rng(seed)
    B, F = fvz.shape[:2]
    nan = np.zeros((B, F, 9), bool)
    pick = rng.uniform(size=(B, F)) < percent / 100.0
    nan[pick, rng.integers(9, size=pick.sum())] = True
    return nan


def scene_c4_shard():
    fvz, fvi, fnz = synthetic.icosphere_views(32, 5, seed=1234, jitter=0.05)
    return case(fvz, fvi, fnz, 1024, 1024, scattered(fvz, 1, 91))


def scene_wide_2048():
    fvz, fvi, fnz = synthetic.icosphere_views(1, 6, seed=92, radius=2.2)
    sliver = np.array([[[[-1.0, -1.0], [1.0, 1.0], [1.0, 0.995]]]], np.float32)   # every tile row, 4 words
    fvi = np.concatenate([fvi, sliver], 1)
    fvz = np.concatenate([fvz, np.full((1, 1, 3), -9.0, np.float32)], 1)
    fnz = np.concatenate([fnz, np.ones((1, 1), np.float32)], 1)
    nan = scattered(fvz, 1, 93)
    nan[0, -1] = False
    return case(fvz, fvi, fnz, 2048, 2048, nan)


SCENES = {**{f"coord_{k}": functools.partial(scene_coord, k) for k in range(10)},
          "bins": scene_bins, "dense": scene_dense, "z_front": scene_z_front, "nan_x": scene_nan_x,
          "culled": scene_culled, "batch_view": scene_batch_view, "all": scene_all,
          "c4_shard": scene_c4_shard, "wide_2048": scene_wide_2048}
BIG = ("c4_shard", "wide_2048")


@functools.lru_cache(maxsize=None)
def scene(name):
    return SCENES[name]()


def tainted_inputs(sc):
    """(fvz, fvi) with NaN in the marked coordinates."""
    fvz, fvi = sc.fvz.copy(), sc.fvi.copy()
    B, F = sc.nan.shape[:2]
    fvz[sc.nan[..., :3]] = np.nan
    fvi.reshape(B, F, 6)[sc.nan[..., 3:]] = np.nan
    return fvz, fvi


def bad(sc):
    return sc.nan.any(-1)


@functools.lru_cache(maxsize=None)
def stripped(name):
    """The scene without its tainted faces -> (fvz, fvi, fnz, keep (B, F) original index of each slot or
    -1 for a filler, slot (B, F) the stripped slot of each original face or -1)."""
    sc = scene(name)
    B, F = sc.fnz.shape
    keep = np.full((B, F), -1, np.int64)
    slot = np.full((B, F), -1, np.int64)
    fvz = np.full_like(sc.fvz, -1.0)
    fvi = np.zeros_like(sc.fvi)
    fvi[..., 0] = OFF
    fnz = np.ones_like(sc.fnz)
    for b in range(B):
        k = np.nonzero(~bad(sc)[b])[0]
        keep[b, :len(k)] = k
        slot[b, k] = np.arange(len(k))
        fvz[b, :len(k)], fvi[b, :len(k)], fnz[b, :len(k)] = sc.fvz[b, k], sc.fvi[b, k], sc.fnz[b, k]
    return fvz, fvi, fnz, keep, slot


def strip_faces(name, a):
    """Per-face array (B, F, ...) of the tainted scene -> the stripped scene's (fillers: zeros)."""
    _, _, _, keep, _ = stripped(name)
    out = np.zeros_like(a)
    for b in range(a.shape[0]):
        n = (keep[b] >= 0).sum()
        out[b, :n] = a[b, keep[b, :n]]
    return out


def unstrip_faces(name, a):
    """Per-face array of the stripped scene -> the tainted scene's layout, tainted rows zero."""
    _, _, _, keep, _ = stripped(name)
    out = np.zeros_like(a)
    for b in range(a.shape[0]):
        n = (keep[b] >= 0).sum()
        out[b, keep[b, :n]] = a[b, :n]
    return out


def map_idx(name, idx):
    """Stripped face_idx -> original indices."""
    keep = torch.from_numpy(stripped(name)[3]).to(idx.device)
    b = torch.arange(idx.shape[0], device=idx.device).view(-1, 1, 1).expand_as(idx)
    return torch.where(idx >= 0, keep[b, idx.clamp(min=0)], idx)


# ---------------------------------------------------------------------------------------------------
def T(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    return t if dtype is None else t.to(dtype)


def N(t):
    return t.detach().float().cpu().numpy() if t.dtype == torch.bfloat16 else t.detach().cpu().numpy()


def bits(t):
    t = t.detach()
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int64 if t.element_size() == 8 else torch.int32)


def same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(bits(a), bits(b))


@functools.lru_cache(maxsize=None)
def grads_out(name, D=3):
    sc = scene(name)
    B, F = sc.fnz.shape
    rng = np.random.default_rng(95)
    return (synthetic.random_features(B, F, D, seed=96),
            rng.random((B, sc.H, sc.W, D), dtype=np.float32) * 2 - 1,
            rng.random((B, sc.H, sc.W), dtype=np.float32) * 2 - 1)


def traced(fn):
    _lib.trace_begin()
    try:
        out = fn()
    finally:
        ran = [k for k, _ in _lib.trace_end()]
    return out, ran


def fused(name, strip, dtype="fp32", knum=30, outs=("feat", "soft"), views=False):
    """dibr_rasterization on the tainted (strip False) or stripped scene, and its backward through the
    outputs `outs` -> dict of outputs (gradients in the tainted scene's layout) and the forward's kernels."""
    from kaolin_b200.render.mesh import _host, dibr_rasterization
    sc = scene(name)
    ff, g_feat, g_soft = grads_out(name)
    if strip:
        fvz, fvi, fnz, _, _ = stripped(name)
        ff = strip_faces(name, ff)
    else:
        (fvz, fvi), fnz = tainted_inputs(sc), sc.fnz
    real = torch.float64 if dtype == "f64" else torch.float32
    fdt = {"fp32": torch.float32, "bf16": torch.bfloat16, "f64": torch.float64}[dtype]
    t_fvi = T(fvi, real).requires_grad_(bool(outs))
    t_ff = T(ff, fdt).requires_grad_(bool(outs))
    g_feat = T(g_feat, fdt)
    g_soft = T(g_soft, real)
    if views:
        t_fvz, t_fnz = T(fvz), T(fnz)
        feat, idx, wts, soft, ws = _host.forward(_lib.RASTER | _lib.SOFT_MASK, sc.H, sc.W, t_fvz, t_fvi.detach(),
                                                 t_ff.detach(), t_fnz, None, sc.m, EPS, SIGMAINV, sc.boxlen * sc.m, knum)
        B = fvz.shape[0]
        g_fvi = torch.empty_like(t_fvi)
        g_ff = torch.empty(ff.shape, dtype=torch.float32, device=DEV)
        for c0, c1 in ((0, B // 2), (B // 2, B)):
            _host.backward(sc.H, sc.W, g_feat, g_soft, idx, wts, soft, t_fvi.detach(), t_ff.detach(), sc.m, EPS,
                           SIGMAINV, sc.boxlen * sc.m, knum, ws, True, views=(c0, c1), out=(g_fvi, g_ff))
        ran = []
    else:
        (feat, soft, idx), ran = traced(lambda: dibr_rasterization(
            sc.H, sc.W, T(fvz, real), t_fvi, t_ff, T(fnz, real), SIGMAINV, sc.boxlen, knum, sc.m, EPS))
        if outs:
            pairs = [(t, g) for k, t, g in (("feat", feat, g_feat), ("soft", soft, g_soft)) if k in outs]
            torch.autograd.backward([p[0] for p in pairs], [p[1] for p in pairs])
        g_fvi, g_ff = t_fvi.grad, t_ff.grad
    out = dict(feat=feat, soft=soft, idx=map_idx(name, idx) if strip else idx)
    if outs or views:
        gf, gff = N(g_fvi).astype(np.float64), N(g_ff).astype(np.float64)
        out.update(g_fvi=unstrip_faces(name, gf) if strip else gf, g_ff=unstrip_faces(name, gff) if strip else gff)
    return out, ran


def rel(a, b):
    scale = max(float(np.abs(b).max()), 1e-30)
    return float(np.abs(a - b).max()) / scale


def assert_absent(name, got, want, what="", ff_tol=SELF_TOL):
    """got (tainted scene) against want (stripped scene, mapped back): images bit-equal, gradients within
    SELF_TOL of scale (ff_tol for grad_face_features) and exactly zero on the tainted faces' rows."""
    sc = scene(name)
    for k in ("idx", "feat", "soft"):
        assert same(got[k], want[k]), (what, k)
    B, F = sc.fnz.shape
    tb = torch.from_numpy(bad(sc)).to(DEV).view(-1)
    idx = got["idx"]
    won = tb[idx.clamp(min=0) + torch.arange(B, device=DEV).view(-1, 1, 1) * F] & (idx >= 0)
    assert not won.any(), (what, "a tainted face wins")
    assert torch.isfinite(got["feat"].float()).all() and torch.isfinite(got["soft"]).all()
    if "g_fvi" in got:
        m = bad(sc)
        for k, tol in (("g_fvi", SELF_TOL), ("g_ff", ff_tol)):
            g = got[k]
            assert np.isfinite(g).all(), (what, k)
            assert (g[m] == 0).all(), (what, k, "tainted rows")
            if np.abs(want[k]).max() > 0:
                assert rel(g, want[k]) <= tol, (what, k, rel(g, want[k]))
            else:
                assert (g == 0).all(), (what, k)


SMALL = [n for n in SCENES if n not in BIG]


# ---------------------------------------------------------------------------------------------------
# (a) the library on the stripped scene
@pytest.mark.parametrize("dtype,knum", [("fp32", 30), ("fp32", 100), ("bf16", 30), ("f64", 30)])
@pytest.mark.parametrize("name", SMALL)
def test_fused_equals_stripped_scene(name, dtype, knum):
    got, ran = fused(name, False, dtype, knum)
    want, ran_s = fused(name, True, dtype, knum)
    assert ran == ran_s, (ran, ran_s)
    assert_absent(name, got, want, f"{dtype} k{knum}", BF16_TOL if dtype == "bf16" else SELF_TOL)
    if name == "all":
        assert (got["idx"] == -1).all() and (got["soft"] == 0).all() and (got["g_fvi"] == 0).all()


@pytest.mark.parametrize("outs", [("feat",), ("soft",)])
@pytest.mark.parametrize("name", ["coord_9", "bins", "dense", "z_front", "culled"])
def test_backward_through_one_output(name, outs):
    got, _ = fused(name, False, outs=outs)
    want, _ = fused(name, True, outs=outs)
    assert_absent(name, got, want, outs[0])


@pytest.mark.parametrize("name", ["coord_9", "bins", "dense", "z_front", "culled", "batch_view"])
def test_cache_and_recompute_backward(name, monkeypatch):
    """No hit cache: every soft-mask tile is recomputed in backward; a full cache is the default."""
    from kaolin_b200.render.mesh import _host
    monkeypatch.setattr(_host, "CACHE_TILE_FRACTION", 0.0)
    monkeypatch.setattr(_host, "CACHE_MIN_TILES", 1)
    got, _ = fused(name, False)
    want, _ = fused(name, True)
    assert_absent(name, got, want, "recompute")


@pytest.mark.parametrize("name", ["dense", "culled", "batch_view", "all"])
def test_view_chunked_backward(name):
    got, _ = fused(name, False, views=True)
    want, _ = fused(name, True, views=True)
    assert_absent(name, got, want, "views")


@pytest.mark.parametrize("dtype", ["fp32", "f64"])
@pytest.mark.parametrize("name", ["coord_9", "bins", "dense", "z_front", "culled", "batch_view", "all"])
def test_rasterize_and_soft_mask_alone(name, dtype):
    """rasterize with and without valid_faces, then dibr_soft_mask on its face_idx, with backward; a
    caller's face_idx that points at a tainted face still counts as covered."""
    from kaolin_b200.render.mesh import dibr_soft_mask, rasterize
    sc = scene(name)
    ff, g_feat, g_soft = grads_out(name)
    real = torch.float64 if dtype == "f64" else torch.float32
    (fvz, fvi), fnz = tainted_inputs(sc), sc.fnz
    s_fvz, s_fvi, s_fnz, _, _ = stripped(name)
    s_ff = strip_faces(name, ff)
    valid = fnz >= 0
    valid[..., 1::3] = False
    s_valid = strip_faces(name, valid)
    for v, sv in ((None, None), (valid, s_valid)):
        res = []
        for z, xy, f, vv in ((fvz, fvi, ff, v), (s_fvz, s_fvi, s_ff, sv)):
            a_fvi, a_ff = T(xy, real).requires_grad_(), T(f, real).requires_grad_()
            feat, idx = rasterize(sc.H, sc.W, T(z, real), a_fvi, a_ff, None if vv is None else T(vv), sc.m, EPS)
            feat.backward(T(g_feat, real))
            res.append((feat, idx, N(a_fvi.grad), N(a_ff.grad)))
        (feat, idx, gx, gf), (s_feat, s_idx, s_gx, s_gf) = res
        assert same(feat, s_feat) and torch.equal(idx, map_idx(name, s_idx))
        for g, sg in ((gx, s_gx), (gf, s_gf)):
            sg = unstrip_faces(name, sg)
            assert (g[bad(sc)] == 0).all() and np.isfinite(g).all()
            assert rel(g, sg) <= SELF_TOL if np.abs(sg).max() > 0 else (g == 0).all()
    # dibr_soft_mask alone sees face_vertices_image only: a face is tainted there by a NaN in it, and the
    # scene without such faces is the same one with them moved off screen (the order of the others is
    # kept).  Coverage comes only from the sign of face_idx, so both calls take the same one, here with
    # a tainted face's index on some pixels.
    idx = idx.clone()
    tb = np.nonzero(bad(sc)[0])[0]
    if len(tb):
        idx[0, ::7, ::5] = int(tb[0])
    xy_bad = sc.nan[..., 3:].any(-1)
    s_fvi = fvi.copy()
    s_fvi[xy_bad] = 0.0
    s_fvi[xy_bad, :, 0] = OFF
    res = []
    for xy in (fvi, s_fvi):
        a_fvi = T(xy, real).requires_grad_()
        soft = dibr_soft_mask(a_fvi, idx, SIGMAINV, sc.boxlen, 30, sc.m)
        soft.backward(T(g_soft, real))
        res.append((soft, N(a_fvi.grad)))
    (soft, gx), (s_soft, s_gx) = res
    assert same(soft, s_soft)
    if len(tb):
        assert (soft[0, ::7, ::5] == 1).all()
    assert (gx[xy_bad] == 0).all() and (s_gx[xy_bad] == 0).all() and np.isfinite(gx).all()
    assert rel(gx, s_gx) <= SELF_TOL if np.abs(s_gx).max() > 0 else (gx == 0).all()


def test_batch_view_neighbours_unchanged():
    """The fully tainted view is empty; views 0 and 2 are bit-identical to a batch of those two alone."""
    from kaolin_b200.render.mesh import dibr_rasterization
    name = "batch_view"
    sc = scene(name)
    got, _ = fused(name, False)
    assert (got["idx"][1] == -1).all() and (got["soft"][1] == 0).all() and (got["feat"][1] == 0).all()
    assert (got["g_fvi"][1] == 0).all() and (got["g_ff"][1] == 0).all()
    ff, g_feat, g_soft = grads_out(name)
    k = [0, 2]
    a_fvi, a_ff = T(sc.fvi[k]).requires_grad_(), T(ff[k]).requires_grad_()
    feat, soft, idx = dibr_rasterization(sc.H, sc.W, T(sc.fvz[k]), a_fvi, a_ff, T(sc.fnz[k]),
                                         SIGMAINV, sc.boxlen, 30, sc.m, EPS)
    torch.autograd.backward([feat, soft], [T(g_feat[k]), T(g_soft[k])])
    assert same(feat, got["feat"][k]) and same(soft, got["soft"][k]) and torch.equal(idx, got["idx"][k])
    assert rel(got["g_fvi"][k], N(a_fvi.grad)) <= SELF_TOL and rel(got["g_ff"][k], N(a_ff.grad)) <= SELF_TOL


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("name", BIG)
def test_large_scenes(name, dtype):
    """1 % tainted at bench.py's shape and at 2048^2: the persistent forward, the fused soft-mask forward,
    and the hit-cache backward."""
    sc = scene(name)
    got, ran = fused(name, False, dtype)
    if name == "c4_shard":
        assert "dibr_fwd2_kernel<S=2>" in ran and "soft_fwd_kernel" in ran, ran
    want, ran_s = fused(name, True, dtype)
    assert ran == ran_s
    assert_absent(name, got, want, dtype, BF16_TOL if dtype == "bf16" else SELF_TOL)
    assert (got["idx"] >= 0).any() and bad(sc).sum() > 10 * sc.fnz.shape[0]


def test_large_scene_recompute_backward(monkeypatch):
    from kaolin_b200.render.mesh import _host
    monkeypatch.setattr(_host, "CACHE_TILE_FRACTION", 0.0)
    monkeypatch.setattr(_host, "CACHE_MIN_TILES", 64)
    got, _ = fused("wide_2048", False)
    want, _ = fused("wide_2048", True)
    assert_absent("wide_2048", got, want, "recompute")


def test_graphed_call():
    from kaolin_b200.render.mesh import dibr_rasterization, make_graphed_dibr_rasterization
    name = "culled"
    sc = scene(name)
    ff, g_feat, g_soft = grads_out(name)
    fvz, fvi = tainted_inputs(sc)
    f = make_graphed_dibr_rasterization(sc.H, sc.W, T(sc.fvz), T(sc.fvi).requires_grad_(), T(ff).requires_grad_(),
                                        T(sc.fnz), SIGMAINV, sc.boxlen, 30, sc.m, EPS)
    a_fvi, a_ff = T(fvi).requires_grad_(), T(ff).requires_grad_()
    feat, soft, idx = f(T(fvz), a_fvi, a_ff, T(sc.fnz))
    torch.autograd.backward([feat, soft], [T(g_feat), T(g_soft)])
    got = dict(feat=feat.clone(), soft=soft.clone(), idx=idx.clone(),
               g_fvi=N(a_fvi.grad).astype(np.float64), g_ff=N(a_ff.grad).astype(np.float64))
    want, _ = fused(name, True)
    assert_absent(name, got, want, "graphed")


def test_reruns_no_sync_no_stderr(capfd):
    """Byte-identical reruns, no host synchronisation in the forward or the backward, nothing on stderr."""
    from kaolin_b200.render.mesh import dibr_rasterization
    name = "bins"
    sc = scene(name)
    ff, g_feat, g_soft = grads_out(name)
    fvz, fvi = tainted_inputs(sc)
    args = [T(x) for x in (fvz, fvi, ff, sc.fnz, g_feat, g_soft)]
    torch.cuda.synchronize()
    capfd.readouterr()
    outs = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(2):
            a_fvi, a_ff = args[1].clone().requires_grad_(), args[2].clone().requires_grad_()
            feat, soft, idx = dibr_rasterization(sc.H, sc.W, args[0], a_fvi, a_ff, args[3], SIGMAINV, sc.boxlen, 30,
                                                 sc.m, EPS)
            torch.autograd.backward([feat, soft], [args[4], args[5]])
            outs.append((feat, soft, idx))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    (a, b, c), (d, e, f) = outs
    assert same(a, d) and same(b, e) and torch.equal(c, f)
    assert capfd.readouterr().err == ""


# ---------------------------------------------------------------------------------------------------
# (b) the reference's kernels and (c) the C oracle, on the stripped scene
def reference_stripped(name, dtype="fp32", knum=30):
    sc = scene(name)
    ff, g_feat, g_soft = grads_out(name)
    fvz, fvi, fnz, _, _ = stripped(name)
    ff = strip_faces(name, ff)
    if dtype == "bf16":
        ff = T(ff, torch.bfloat16).float()
        g_feat = T(g_feat, torch.bfloat16).float()
    else:
        ff, g_feat = T(ff), T(g_feat)

    def live():
        out = ref_cuda.dibr_forward_backward(sc.H, sc.W, T(fvz), T(fvi), ff, T(fnz), g_feat, T(g_soft),
                                             SIGMAINV, sc.boxlen, knum, sc.m, EPS)
        out["face_idx"] = map_idx(name, out["face_idx"])
        out["features_bf16"] = out["features"].to(torch.bfloat16)
        out["grad_fvi"] = torch.from_numpy(unstrip_faces(name, N(out["grad_fvi"])))
        out["grad_ff"] = torch.from_numpy(unstrip_faces(name, N(out["grad_ff"])))
        return out

    names = ("face_idx", "features_bf16" if dtype == "bf16" else "features", "soft_mask", "grad_fvi", "grad_ff")
    return ref_golden.reference(f"nan_{name}_{dtype}_k{knum}", live, names=names, path=STORE, sample_rows=64,
                                digest_only=("face_idx", "features", "features_bf16", "soft_mask"))


REF_CASES = [(n, "fp32", 30) for n in SCENES] + [(n, "fp32", 100) for n in SMALL] + \
            [(n, "bf16", 30) for n in ("coord_9", "bins", "dense", "c4_shard")]


@pytest.mark.parametrize("name,dtype,knum", REF_CASES, ids=[f"{n}-{d}-k{k}" for n, d, k in REF_CASES])
def test_tainted_scene_is_the_reference_on_the_stripped_scene(name, dtype, knum):
    r = reference_stripped(name, dtype, knum)
    got, _ = fused(name, False, dtype, knum)
    assert r.equal("face_idx", got["idx"]) and r.equal("soft_mask", got["soft"])
    assert r.equal("features_bf16" if dtype == "bf16" else "features", got["feat"])
    tol = BF16_TOL if dtype == "bf16" else GRAD_TOL
    for k, ours in (("grad_fvi", "g_fvi"), ("grad_ff", "g_ff")):
        if dtype == "bf16" and k == "grad_fvi":
            continue
        a, b = r.pair(k, got[ours])
        assert float(np.abs(a - b).max()) <= tol * max(r.scale(k), 1e-30), k


ORACLE_CASES = [(n, k) for n in SMALL for k in (30, 100)]


@pytest.mark.parametrize("name,knum", ORACLE_CASES, ids=[f"{n}-k{k}" for n, k in ORACLE_CASES])
def test_gradients_against_c_oracle(name, knum):
    sc = scene(name)
    if sc.fnz.size * sc.H * sc.W > ORACLE_MAX_WORK:
        pytest.skip("too large for the brute-force oracle")
    ff, g_feat, g_soft = grads_out(name)
    fvz, fvi, fnz, _, _ = stripped(name)
    s_ff = strip_faces(name, ff)
    _, _, idx, w = oracle.dibr_rasterization(sc.H, sc.W, fvz, fvi, s_ff, fnz, SIGMAINV, sc.boxlen, knum, sc.m, EPS,
                                             return_weights=True)
    o_gx, o_gf, _, _ = oracle.dibr_rasterization_backward(g_feat, g_soft, idx, w, fvi, s_ff, SIGMAINV, sc.boxlen,
                                                          knum, sc.m, EPS)
    got, _ = fused(name, False, "fp32", knum)
    assert torch.equal(got["idx"], map_idx(name, T(idx)))
    for k, o in (("g_fvi", o_gx), ("g_ff", o_gf)):
        o = unstrip_faces(name, o.astype(np.float64))
        if np.abs(o).max() == 0:
            assert (got[k] == 0).all()
        else:
            assert rel(got[k], o) <= GRAD_TOL, k


# ---------------------------------------------------------------------------------------------------
# the deviation: the reference on the tainted scene
@pytest.mark.parametrize("name", ["z_front", "nan_x"])
def test_reference_differs_where_a_tainted_face_wins(name):
    sc = scene(name)
    ff, _, _ = grads_out(name)
    fvz, fvi = tainted_inputs(sc)

    def live():
        _, idx, _ = ref_cuda.rasterize_forward(sc.H, sc.W, T(fvz), T(fvi), T(ff), T(sc.fnz) >= 0, sc.m, EPS)
        return {"face_idx": idx}

    r = ref_golden.reference(f"nan_deviation_{name}", live, names=("face_idx",), full=("face_idx",), path=STORE)
    ref_idx = r.pair("face_idx", torch.zeros((1, sc.H, sc.W), dtype=torch.int64))[1].reshape(1, sc.H, sc.W)
    got, _ = fused(name, False, outs=())
    ours = N(got["idx"])
    tainted = np.nonzero(bad(sc)[0])[0]
    wins = np.isin(ref_idx, tainted)
    assert wins.sum() > 20, wins.sum()
    assert (ours[wins] != ref_idx[wins]).all()
    assert not np.isin(ours, tainted).any()
