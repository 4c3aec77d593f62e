"""The fused rasterize backward recomputes the barycentric weights when it is given none.

A forward through the C ABI that also writes the weights, then the backward once with those
weights and once with NULL (the kernels recompute them from face_idx, the vertices times the
multiplier, and eps).  The recomputed weights are the forward's bits, so the two gradients may
differ only by the order of the float atomics.  That spread is measured here by running the
backward with weights twice (1.3e-7 of the gradient's scale for fp32 D = 1 on an H100; at
c4_shard two runs of the same build differ by up to 3.3e-7).  The bound below (1e-6) is the one
the other backward-equivalence tests use.
"""
import numpy as np
import pytest
import torch

from kaolin_b200 import _lib, synthetic
from kaolin_b200.render.mesh import _host

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SIGMAINV, BOXLEN_M, KNUM = 7000., 20., 30


def forward_with_weights(H, W, fvz, fvi, ff, fnz, multiplier, eps):
    B, F = fvi.shape[:2]
    D = ff.shape[-1]
    bf16 = ff.dtype == torch.bfloat16
    feat = torch.empty((B, H, W, D), dtype=ff.dtype, device=DEV)
    idx = torch.empty((B, H, W), dtype=torch.int64, device=DEV)
    wts = torch.empty((B, H, W, 3), dtype=torch.float32, device=DEV)
    soft = torch.empty((B, H, W), dtype=torch.float32, device=DEV)
    ws = _host.workspace(B, B * F, H, W, DEV, KNUM)
    fn = _lib.lib().dibr_b200_forward_bf16 if bf16 else _lib.lib().dibr_b200_forward
    p = _host.ptr
    st = fn(B, F, H, W, D, p(fvz), p(fvi), p(ff), p(fnz), None, float(multiplier), float(eps), 3, SIGMAINV,
            BOXLEN_M, KNUM, p(feat), p(idx), p(wts), p(soft), p(ws), ws.numel(), _host.stream_ptr(DEV))
    _lib.check(st, "dibr_b200_forward")
    return feat, idx, wts, soft, ws


def rel(a, b):
    a, b = a.float().cpu().numpy(), b.float().cpu().numpy()
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


CASES = [  # (id, D, dtype, W, multiplier); D > 4 or a width that is not a multiple of 4 selects the warp reduction
    ("rows_D1", 1, torch.float32, 160, 1000.),
    ("rows_D2", 2, torch.float32, 160, 1000.),
    ("rows_D3", 3, torch.float32, 160, 1000.),
    ("rows_D4", 4, torch.float32, 160, 1000.),
    ("rows_D3_mult100", 3, torch.float32, 160, 100.),
    ("rows_bf16_D3", 3, torch.bfloat16, 160, 1000.),
    ("warp_D5", 5, torch.float32, 160, 1000.),
    ("warp_odd_width", 3, torch.float32, 151, 1000.),
    ("warp_odd_width_D1", 1, torch.float32, 151, 1000.),
    ("warp_odd_width_bf16", 2, torch.bfloat16, 151, 1000.),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_backward_without_weights_equals_backward_with_weights(case):
    name, D, dt, W, mult = case
    fvz, fvi, fnz = synthetic.icosphere_views(5, 4, seed=81)
    B, F = fvz.shape[:2]
    H = 144
    t = lambda a: torch.from_numpy(a).to(DEV)
    t_fvz, t_fvi, t_fnz = t(fvz), t(fvi), t(fnz)
    ff = t(synthetic.random_features(B, F, D, seed=82)).to(dt)
    gen = torch.Generator(device=DEV); gen.manual_seed(83)
    g_feat = torch.rand((B, H, W, D), device=DEV, generator=gen).to(dt)
    g_soft = torch.rand((B, H, W), device=DEV, generator=gen)
    feat, idx, wts, soft, ws = forward_with_weights(H, W, t_fvz, t_fvi, ff, t_fnz, mult, 1e-8)
    assert (idx >= 0).float().mean() > 0.05

    # the forward without weights computes the same outputs
    feat2, idx2, none, soft2, _ = _host.forward(3, H, W, t_fvz, t_fvi, ff, t_fnz, None, mult, 1e-8,
                                                SIGMAINV, BOXLEN_M, KNUM)
    assert none is None
    assert torch.equal(idx, idx2) and torch.equal(feat, feat2) and torch.equal(soft, soft2)

    def bwd(w, **kw):
        return _host.backward(H, W, g_feat, g_soft, idx, w, soft, t_fvi, ff, mult, 1e-8, SIGMAINV, BOXLEN_M,
                              KNUM, ws, True, **kw)

    a_fvi, a_ff = bwd(wts)
    b_fvi, b_ff = bwd(wts)
    spread = max(rel(a_fvi, b_fvi), rel(a_ff, b_ff))
    _lib.trace_begin()
    r_fvi, r_ff = bwd(None)
    ran = [k for k, _ in _lib.trace_end()]
    assert ("raster_bwd_rows_kernel" if name.startswith("rows") else "raster_bwd_kernel") in ran, ran
    print(f"[{name}] same backward twice: {spread:.2e}; recomputed vs given: "
          f"fvi {rel(r_fvi, a_fvi):.2e} ff {rel(r_ff, a_ff):.2e}")
    assert rel(r_fvi, a_fvi) <= 1e-6 and rel(r_ff, a_ff) <= 1e-6

    # the two-call split (rasterize branch, hook, soft-mask branch with ACCUMULATE)
    hooked = []
    s_fvi, s_ff = bwd(None, feature_grad_hook=lambda g: hooked.append(g.clone()))
    assert len(hooked) == 1
    assert rel(s_fvi, a_fvi) <= 1e-6 and rel(s_ff, a_ff) <= 1e-6 and rel(hooked[0], a_ff) <= 1e-6

    # view chunks written into shared full-batch buffers
    g_fvi = torch.full_like(t_fvi, float("nan"))
    g_ff = torch.full(ff.shape, float("nan"), dtype=torch.float32, device=DEV)
    for c0, c1 in ((0, 2), (2, 5)):
        bwd(None, views=(c0, c1), out=(g_fvi, g_ff))
    assert rel(g_fvi, a_fvi) <= 1e-6 and rel(g_ff, a_ff) <= 1e-6


def test_rasterize_backward_needs_weights():
    """The operator-level backward follows the packed forward, whose xy is already multiplied:
    it cannot recompute the weights and rejects NULL."""
    B, F, H, W, D = 1, 4, 16, 16, 3
    g = torch.zeros((B, H, W, D), device=DEV)
    idx = torch.full((B, H, W), -1, dtype=torch.int64, device=DEV)
    fvi = torch.zeros((B, F, 3, 2), device=DEV)
    ff = torch.zeros((B, F, 3, D), device=DEV)
    g_fvi = torch.empty_like(fvi)
    g_ff = torch.empty_like(ff)
    p = _host.ptr
    st = _lib.lib().dibr_b200_rasterize_backward(B, F, H, W, D, p(g), p(idx), None, p(fvi), p(ff), 1e-8,
                                                p(g_fvi), p(g_ff), _host.stream_ptr(DEV))
    assert st == _lib.EINVAL
