"""The forward launcher picks one of two tile kernels from the problem shape: dibr_fwd2_kernel (2x2
tiles per CTA) for sparse meshes on large grids (faces per view <= 40 x 32x32 tiles, and 32x32 tiles x
views >= 2048), dibr_tile_fwd_kernel (one tile per CTA) otherwise.  Each test asserts through the
library's per-launch trace which kernel its shape reached, so it fails if the shape stops covering
the path it claims to cover."""
import numpy as np
import pytest
import torch

import oracle
from kaolin_b200 import _lib, synthetic
from kaolin_b200.render.mesh import dibr_rasterization

pytestmark = pytest.mark.gpu
DEV = "cuda"
FWD2, TILE = "dibr_fwd2_kernel<S=2>", "dibr_tile_fwd_kernel"
K_CHUNK = 256   # candidates per staging round of dibr_fwd2_kernel


def traced_forward(H, W, fvz, fvi, ff, fnz, **kw):
    """dibr_rasterization's forward -> (feat, soft, idx, names of the kernels it launched)."""
    _lib.trace_begin()
    feat, soft, idx = dibr_rasterization(H, W, fvz, fvi, ff, fnz, **kw)
    return feat, soft, idx, [name for name, _ in _lib.trace_end()]


def assert_ran(names, kernel):
    other = TILE if kernel == FWD2 else FWD2
    assert kernel in names and other not in names, names


SCENES = {  # name: (generator, H, W, forward kernel the shape selects)
    "ico4_256": (lambda: synthetic.icosphere_views(2, 4, seed=3), 256, 256, TILE),
    "soup2000_200x72": (lambda: synthetic.triangle_soup(1, 2000, seed=5), 200, 72, TILE),  # ~10^2 candidates per tile
    # > 256 candidates per 32x32 tile; 6000 faces >= 32 x 64 16x16 tiles also selects the aggregated binning
    "soup6000_128_dense": (lambda: synthetic.triangle_soup(1, 6000, seed=6, coverage=6.0), 128, 128, TILE),
    # 5120 faces <= 40 x 256 32x32 tiles, and 256 tiles x 8 views >= 2048
    "ico4_512_8views": (lambda: synthetic.icosphere_views(8, 4, seed=3), 512, 512, FWD2),
}


@pytest.mark.parametrize("scene", list(SCENES))
def test_default_selection_equals_oracle(scene):
    gen, H, W, kernel = SCENES[scene]
    fvz, fvi, fnz = gen()
    B, F = fvz.shape[:2]
    ff = synthetic.random_features(B, F, 3, seed=11)
    rng = np.random.default_rng(12)
    g_feat = rng.uniform(size=(B, H, W, 3)).astype(np.float32)
    g_soft = rng.uniform(size=(B, H, W)).astype(np.float32)
    T = lambda a: torch.from_numpy(a).to(DEV)
    t_fvi, t_ff = T(fvi).requires_grad_(True), T(ff).requires_grad_(True)
    feat, soft, idx, ran = traced_forward(H, W, T(fvz), t_fvi, t_ff, T(fnz))
    assert_ran(ran, kernel)
    torch.autograd.backward([feat, soft], [T(g_feat), T(g_soft)])
    o_feat, o_soft, o_idx, o_w = oracle.dibr_rasterization(H, W, fvz, fvi, ff, fnz, return_weights=True)
    assert np.array_equal(idx.cpu().numpy(), o_idx)
    np.testing.assert_allclose(feat.detach().cpu().numpy(), o_feat, rtol=0, atol=1e-5)
    np.testing.assert_allclose(soft.detach().cpu().numpy(), o_soft, rtol=0, atol=1e-5)
    o_gxy, o_gff, _, _ = oracle.dibr_rasterization_backward(g_feat, g_soft, o_idx, o_w, fvi, ff)
    rel = lambda a, b: float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))
    assert rel(t_fvi.grad.cpu().numpy(), o_gxy) <= 3e-5      # vs the double-accumulating CPU oracle
    assert rel(t_ff.grad.cpu().numpy(), o_gff) <= 3e-5


def _random_scene(rng, B, F, kind, spread=1.1):
    """Triangle soups that stress the conservative block culling of dibr_fwd2_kernel: slivers,
    zero-area and duplicated faces, faces larger than the image, vertices far off screen, exact
    depth ties, many faces through one pixel.  Face centres are uniform in [-spread, spread]^2."""
    c = rng.uniform(-spread, spread, (B, F, 1, 2))
    if kind == "tiny":
        off = rng.normal(0, 0.01, (B, F, 3, 2))
    elif kind == "huge":
        off = rng.normal(0, 1.5, (B, F, 3, 2))
    elif kind == "sliver":
        d = rng.normal(0, 0.3, (B, F, 1, 2))
        off = d * rng.uniform(-1, 1, (B, F, 3, 1)) + rng.normal(0, 1e-4, (B, F, 3, 2))
    else:
        off = rng.normal(0, 0.08, (B, F, 3, 2))
    fvi = (c + off).astype(np.float32)
    fvz = rng.uniform(-3, -1, (B, F, 3)).astype(np.float32)
    if kind == "degenerate":
        fvi[:, ::7, 2] = fvi[:, ::7, 1]                 # zero area
        fvi[:, 1::7] = fvi[:, 0::7][:, :fvi[:, 1::7].shape[1]]   # duplicates -> exact depth ties
        fvz[:, 1::7] = fvz[:, 0::7][:, :fvz[:, 1::7].shape[1]]
        fvi[:, 3::11, 0] = 1e4                          # far off screen
    fnz = rng.uniform(-0.2, 1.0, (B, F)).astype(np.float32)
    return fvz, fvi, fnz


def _candidates_of_cta(fvi, fnz, H, W, cx, cy):
    """Valid faces of the first view whose pixel bounding box meets the 32x32 CTA tile (cx, cy)."""
    px = (fvi[0, ..., 0].astype(np.float64) + 1.0) * W / 2 - 0.5
    py = (1.0 - fvi[0, ..., 1].astype(np.float64)) * H / 2 - 0.5
    meets = ((px.max(1) >= 32 * cx) & (px.min(1) < 32 * cx + 32) &
             (py.max(1) >= 32 * cy) & (py.min(1) < 32 * cy + 32))
    return int((meets & (fnz[0] >= 0)).sum())


TRIALS = [  # (H, W, faces per view, multiplier, views, centre spread); F <= 40 x 32x32 tiles, so that
    (96, 128, 450, None, 2, 1.1),   # repeating the views reaches dibr_fwd2_kernel; sizes not multiples of 32
    (77, 203, 800, 1000., 2, 1.1),
    (160, 64, 300, 37.5, 2, 1.1),
    (512, 512, 4000, 1e4, 2, 1.1),
    # 3000 faces centred in a ~48x48 px window: the CTAs there stage more than K_CHUNK candidates in
    # several rounds, while the average per view stays far below the density bound; 1 view: 1024
    # 32x32 tiles (tile kernel), 2 views: 2048 (dibr_fwd2_kernel)
    (1024, 1024, 3000, None, 1, 0.045),
]


@pytest.mark.parametrize("kind", ["mixed", "tiny", "huge", "sliver", "degenerate"])
def test_fwd2_bit_identical_to_tile_kernel(kind):
    """face_idx, features and soft mask of dibr_fwd2_kernel (2x2 tiles per CTA, conservative block culling,
    shared-reciprocal divisions) are BIT-IDENTICAL to dibr_tile_fwd_kernel (per-lane walk over every
    rectangle hit) on adversarial scenes, image sizes that are not multiples of 32 and other multipliers.
    Views are independent in every kernel: the same views rendered at a batch small enough for the tile
    kernel and repeated until the batch selects dibr_fwd2_kernel must give the same bits."""
    rng = np.random.default_rng({"mixed": 1, "tiny": 2, "huge": 3, "sliver": 4, "degenerate": 5}[kind])
    T = lambda a: torch.from_numpy(a).to(DEV)
    for trial, (H, W, F, mult, nv, spread) in enumerate(TRIALS):
        fvz, fvi, fnz = _random_scene(rng, nv, F, kind, spread)
        ff = synthetic.random_features(nv, F, 3, seed=trial)
        tiles32 = ((H + 31) // 32) * ((W + 31) // 32)
        assert F <= 40 * tiles32 and tiles32 * nv < 2048
        reps = -(-2048 // (tiles32 * nv))
        if nv == 1:   # the packed window around pixel (512, 512)
            assert _candidates_of_cta(fvi, fnz, H, W, 15, 15) > K_CHUNK
        rep = lambda a: T(np.concatenate([a] * reps))
        small = traced_forward(H, W, T(fvz), T(fvi), T(ff), T(fnz), multiplier=mult)
        big = traced_forward(H, W, rep(fvz), rep(fvi), rep(ff), rep(fnz), multiplier=mult)
        assert_ran(small[3], TILE)
        assert_ran(big[3], FWD2)
        for i, what in ((2, "face_idx"), (0, "features"), (1, "soft_mask")):
            for r in range(reps):
                assert torch.equal(big[i][r * nv:(r + 1) * nv], small[i]), (kind, trial, r, what)
        if H == 512:   # 4000 faces on 512^2 px: the comparison covers rasterized pixels
            assert (small[2] >= 0).any()
