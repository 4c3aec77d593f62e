"""Every template instantiation of the rasterizer against the oracle.

The launcher picks each kernel from the problem's shape and the feature dtype, never from a user
switch (dibr_b200.cu: launch_fwd, backward_impl, launch_raster_bwd_rows), and each instantiation has its
own staging layout and store path.  So each one is run here and compared with an independent reference,
and each case asserts through the library's per-launch trace which kernel it reached:

a. dibr_fwd2_kernel<SOFT, FT> for D = 1..5 in fp32 and bf16, at a width that is a multiple of 4 and one
   that is not (per-pixel stores instead of the constant-tile vector stores);
b. raster_bwd_rows_kernel<D, FT> for D = 1..4 at strips 4 and 32, D = 3 also at 8 and 16: several
   cp.async-staged slabs per job, a last strip 8 columns wide and a partial last band of rows;
c. raster_bwd_kernel<D, FT> for D = 1..4 and the generic D (odd width);
d. the benchmarked bf16 configuration (bench.py's c4_shard) against its fp32 twin on the upcast inputs.

Inputs that are contiguous views at a one-element storage offset (legal input that the fused entry
points reject as misaligned) give the results of the aligned call.
"""
import functools

import numpy as np
import pytest
import torch

import bench
import oracle
from kaolin_b200 import _lib, synthetic
from kaolin_b200.render.mesh import _host, dibr_rasterization, dibr_soft_mask, rasterize

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
BF16 = torch.bfloat16
SIGMAINV, BOXLEN, KNUM, MULT, EPS = 7000., 0.02, 30, 1000., 1e-8     # the public API's defaults
BOXLEN_M = BOXLEN * MULT
FWD2, TILE = "dibr_fwd2_kernel<S=2>", "dibr_tile_fwd_kernel"
ROWS, WARP = "raster_bwd_rows_kernel", "raster_bwd_kernel"
TOL = 3e-5     # against the double-accumulating oracle, of the gradient's scale (test_parity_gpu.py)
SAME = 1e-6    # the same sums in another order of the float atomics (test_recomputed_weights_gpu.py)
BF16_ROUND = 2.0 ** -8    # relative error of one round-to-nearest to bf16


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def npy(x):
    return x.detach().float().cpu().numpy()


def traced(fn, *args, **kw):
    """-> (fn's result, names of the kernels it launched)."""
    _lib.trace_begin()
    try:
        out = fn(*args, **kw)
    finally:
        ran = [name for name, _ in _lib.trace_end()]
    return out, ran


def assert_grad_close(ours, ref, tol, what):
    """Max-normalised error <= tol AND element-wise allclose(rtol=tol, atol=tol * the gradient's scale)."""
    ours = npy(ours) if isinstance(ours, torch.Tensor) else ours
    ref = npy(ref) if isinstance(ref, torch.Tensor) else ref
    scale = max(float(np.abs(ref).max()), 1e-30)
    e = float(np.abs(ours - ref).max() / scale)
    assert e <= tol, (what, e)
    assert np.allclose(ours, ref, rtol=tol, atol=tol * scale), what


def assert_bf16_rounding_of(ours, ref, what):
    """A bf16 gradient is the fp32 one rounded once (up to the order of the fp32 atomics)."""
    assert ours.dtype == BF16, what
    ref = ref.float()
    err = (ours.float() - ref).abs()
    assert bool((err <= BF16_ROUND * ref.abs() + SAME * ref.abs().max()).all()), (what, float(err.max()))


def selects_fwd2(B, F, H, W):
    """launch_fwd: faces per view <= 40 x (32x32 tiles) and (32x32 tiles) x views >= 2048."""
    tiles32 = -(-H // 32) * -(-W // 32)
    return F <= 40 * tiles32 and tiles32 * B >= 2048


def rows_strip(B, H, W):
    """The strip launch_raster_bwd_rows picks: 32 columns, halved while it is longer than the 4-column
    slab (kRwSlab) and the (view, 32-row band, strip) jobs number fewer than 8192."""
    strip = 32
    while strip > 4 and B * -(-H // 32) * -(-W // strip) < 8192:
        strip //= 2
    return strip


def forward_with_weights(H, W, fvz, fvi, ff, fnz):
    """The fused forward (rasterize + soft mask) through the C ABI, also writing the weights."""
    B, F = fvi.shape[:2]
    D = ff.shape[-1]
    feat = torch.empty((B, H, W, D), dtype=ff.dtype, device=DEV)
    idx = torch.empty((B, H, W), dtype=torch.int64, device=DEV)
    wts = torch.empty((B, H, W, 3), dtype=torch.float32, device=DEV)
    soft = torch.empty((B, H, W), dtype=torch.float32, device=DEV)
    ws = _host.workspace(B, B * F, H, W, DEV, KNUM)
    fn = _lib.lib().dibr_b200_forward_bf16 if ff.dtype == BF16 else _lib.lib().dibr_b200_forward
    p = _host.ptr
    st = fn(B, F, H, W, D, p(fvz), p(fvi), p(ff), p(fnz), None, MULT, EPS, _lib.RASTER | _lib.SOFT_MASK, SIGMAINV,
            BOXLEN_M, KNUM, p(feat), p(idx), p(wts), p(soft), p(ws), ws.numel(), _host.stream_ptr(DEV))
    _lib.check(st, "dibr_b200_forward")
    return feat, idx, wts, soft, ws


# ---------------------------------------------------------------------------------------------------
# a. forward on dibr_fwd2_kernel
FWD_H = 256


@functools.lru_cache(maxsize=1)
def fwd_scene():
    """32 views of a level-3 icosphere (1 280 faces) and 5 feature channels; D < 5 takes the first D."""
    fvz, fvi, fnz = synthetic.icosphere_views(32, 3, seed=21)
    return fvz, fvi, fnz, synthetic.random_features(32, fvz.shape[1], 5, seed=22)


@functools.lru_cache(maxsize=2)
def fwd_oracle(W):
    """The oracle on views 0-1 (every kernel renders the views independently)."""
    fvz, fvi, fnz, ff = fwd_scene()
    return oracle.dibr_rasterization(FWD_H, W, fvz[:2], fvi[:2], ff[:2], fnz[:2])


@pytest.mark.parametrize("W", [256, 252])
@pytest.mark.parametrize("D", [1, 2, 3, 4, 5])
def test_fwd2_forward(D, W):
    H = FWD_H
    fvz, fvi, fnz, ff5 = fwd_scene()
    B, F = fvz.shape[:2]
    assert selects_fwd2(B, F, H, W) and not selects_fwd2(8, F, H, W)
    t_fvz, t_fvi, t_fnz, t_ff = t(fvz), t(fvi), t(fnz), t(ff5[..., :D])
    valid = t_fnz >= 0

    (feat, soft, idx), ran = traced(dibr_rasterization, H, W, t_fvz, t_fvi, t_ff, t_fnz)
    assert FWD2 in ran and TILE not in ran, ran
    o_feat, o_soft, o_idx = fwd_oracle(W)
    assert (o_idx >= 0).mean() > 0.1
    assert np.array_equal(idx[:2].cpu().numpy(), o_idx)
    np.testing.assert_allclose(npy(feat[:2]), o_feat[..., :D], rtol=0, atol=1e-5)
    np.testing.assert_allclose(npy(soft[:2]), o_soft, rtol=0, atol=1e-5)

    # every view bit-identical to dibr_tile_fwd_kernel, which 8 views at a time select
    for v in range(0, B, 8):
        s = slice(v, v + 8)
        (c_feat, c_soft, c_idx), ran = traced(dibr_rasterization, H, W, t_fvz[s], t_fvi[s], t_ff[s], t_fnz[s])
        assert TILE in ran and FWD2 not in ran, ran
        assert torch.equal(c_idx, idx[s]) and torch.equal(c_feat, feat[s]) and torch.equal(c_soft, soft[s]), v

    # rasterize alone runs dibr_fwd2_kernel<SOFT = false>
    (r_feat, r_idx), ran = traced(rasterize, H, W, t_fvz, t_fvi, t_ff, valid_faces=valid)
    assert FWD2 in ran and not any("soft" in k for k in ran), ran
    assert torch.equal(r_feat, feat) and torch.equal(r_idx, idx)

    # bf16 features: the fp32 arithmetic on the upcast values, rounded to nearest-even once on store
    ff16 = t_ff.to(BF16)
    (b_feat, b_soft, b_idx), ran = traced(dibr_rasterization, H, W, t_fvz, t_fvi, ff16, t_fnz)
    assert FWD2 in ran and TILE not in ran, ran
    u_feat, u_soft, u_idx = dibr_rasterization(H, W, t_fvz, t_fvi, ff16.float(), t_fnz)
    assert b_feat.dtype == BF16
    assert torch.equal(b_idx, u_idx) and torch.equal(b_soft, u_soft)
    assert torch.equal(b_feat, u_feat.to(BF16))
    (rb_feat, rb_idx), ran = traced(rasterize, H, W, t_fvz, t_fvi, ff16, valid_faces=valid)
    assert FWD2 in ran and not any("soft" in k for k in ran), ran
    assert torch.equal(rb_feat, b_feat) and torch.equal(rb_idx, b_idx)


# ---------------------------------------------------------------------------------------------------
# b. / c. rasterize backward: the row walk and the warp reduction
ROWS_H, ROWS_W = 500, 520   # 16 bands of 32 rows, the last one 20; 520 = 16 x 32 + 8 = 32 x 16 + 8 columns
VIEWS_FOR_STRIP = {32: 32, 16: 16, 8: 8, 4: 2}
ROW_CASES = [(D, ft, strip) for ft in ("fp32", "bf16") for D in (1, 2, 3, 4)
             for strip in ((4, 8, 16, 32) if D == 3 else (4, 32))]
WARP_H, WARP_W = 144, 151   # odd width: the warp-reduction kernel for every D


@functools.lru_cache(maxsize=1)
def bwd_scene():
    """32 views of a level-4 icosphere (5 120 faces); a case with B views takes the first B."""
    return synthetic.icosphere_views(32, 4, seed=31)


@functools.lru_cache(maxsize=2)
def oracle_geometry(B, H, W):
    """The oracle's own face_idx and weights for the first B views."""
    fvz, fvi, fnz = (a[:B] for a in bwd_scene())
    _, idx, w = oracle.rasterize(H, W, fvz, fvi, np.zeros(fvz.shape + (1,), np.float32), valid_faces=fnz >= 0,
                                 return_weights=True)
    return idx, w


def check_backward(B, H, W, D, ft, kernel, own_geometry):
    """Forward through the C ABI with stored weights, the production backward (weights recomputed)
    traced to ``kernel``, then the oracle's double-accumulating backward on the same pixels: the
    forward's face_idx and weights, or with ``own_geometry`` the oracle's (and the forward's face_idx
    must equal them).  Then the public API's gradients equal the C ABI's up to the atomics' order and,
    for bf16 features, one rounding."""
    fvz, fvi, fnz = (a[:B] for a in bwd_scene())
    F = fvz.shape[1]
    dt = BF16 if ft == "bf16" else torch.float32
    t_fvz, t_fvi, t_fnz = t(fvz), t(fvi), t(fnz)
    ff = t(synthetic.random_features(B, F, D, seed=40 + D)).to(dt)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(50 + D)
    g = torch.rand((B, H, W, D), device=DEV, generator=gen).to(dt)
    feat, idx, wts, _, ws = forward_with_weights(H, W, t_fvz, t_fvi, ff, t_fnz)
    (g_fvi, g_ff), ran = traced(_host.backward, H, W, g, None, idx, None, None, t_fvi, ff, MULT, EPS, SIGMAINV,
                                BOXLEN_M, KNUM, ws, True)
    other = WARP if kernel == ROWS else ROWS
    assert kernel in ran and other not in ran, ran
    assert g_ff.dtype == torch.float32
    idx_np, w_np = idx.cpu().numpy(), npy(wts)
    assert (idx_np >= 0).mean() > 0.05
    if own_geometry:
        o_idx, w_np = oracle_geometry(B, H, W)
        assert np.array_equal(idx_np, o_idx)
    o_gxy, o_gff = oracle.rasterize_backward(npy(g), idx_np, w_np, fvi, npy(ff))
    assert_grad_close(g_fvi, o_gxy, TOL, "grad_face_vertices_image")
    assert_grad_close(g_ff, o_gff, TOL, "grad_face_features")

    p_fvi, p_ff = t_fvi.clone().requires_grad_(True), ff.clone().requires_grad_(True)
    p_feat, _ = rasterize(H, W, t_fvz, p_fvi, p_ff, valid_faces=t_fnz >= 0)
    assert torch.equal(p_feat, feat)
    p_feat.backward(g)
    assert_grad_close(p_fvi.grad, g_fvi, SAME, "public grad_face_vertices_image")
    if ft == "bf16":
        assert_bf16_rounding_of(p_ff.grad, g_ff, "public grad_face_features")
    else:
        assert_grad_close(p_ff.grad, g_ff, SAME, "public grad_face_features")


@pytest.mark.parametrize("D,ft,strip", ROW_CASES, ids=[f"D{d}-{ft}-strip{s}" for d, ft, s in ROW_CASES])
def test_rows_backward(D, ft, strip):
    B = VIEWS_FOR_STRIP[strip]
    assert rows_strip(B, ROWS_H, ROWS_W) == strip
    check_backward(B, ROWS_H, ROWS_W, D, ft, ROWS, own_geometry=strip == 4)


@pytest.mark.parametrize("ft", ["fp32", "bf16"])
@pytest.mark.parametrize("D", [1, 2, 3, 4, 5])
def test_warp_backward(D, ft):
    check_backward(2, WARP_H, WARP_W, D, ft, WARP, own_geometry=True)


# ---------------------------------------------------------------------------------------------------
# d. BASELINE configs[3] as bench.py --features bf16 runs it
def test_benchmarked_bf16_configuration():
    B, F, H, W, D, fvz, fvi, fnz, ff = bench.make_scene("c4_shard", 0)
    assert selects_fwd2(B, F, H, W) and rows_strip(B, H, W) == 32
    t_fvz, t_fvi, t_fnz = t(fvz), t(fvi), t(fnz)
    ff16 = torch.from_numpy(ff).to(BF16).to(DEV)          # as bench.py casts them
    gen = torch.Generator(device=DEV)
    gen.manual_seed(4321)
    g16 = torch.rand((B, H, W, D), device=DEV, generator=gen).to(BF16)
    g_soft = torch.rand((B, H, W), device=DEV, generator=gen)

    def fused(ff_, g_):
        (feat, idx, _, soft, ws), f_ran = traced(_host.forward, _lib.RASTER | _lib.SOFT_MASK, H, W, t_fvz, t_fvi,
                                                 ff_, t_fnz, None, MULT, EPS, SIGMAINV, BOXLEN_M, KNUM)
        (g_fvi, g_ff), b_ran = traced(_host.backward, H, W, g_, g_soft, idx, None, soft, t_fvi, ff_, MULT, EPS,
                                      SIGMAINV, BOXLEN_M, KNUM, ws, True)
        return feat, idx, soft, g_fvi, g_ff, f_ran + b_ran

    feat, idx, soft, g_fvi, g_ff, ran = fused(ff16, g16)
    for kernel in (FWD2, "soft_fwd_kernel", ROWS, "soft_bwd_runs_kernel"):
        assert kernel in ran, (kernel, ran)
    u_feat, u_idx, u_soft, u_fvi, u_ff, _ = fused(ff16.float(), g16.float())
    assert torch.equal(idx, u_idx) and torch.equal(soft, u_soft) and torch.equal(feat, u_feat.to(BF16))
    assert_grad_close(g_fvi, u_fvi, SAME, "grad_face_vertices_image")
    assert_grad_close(g_ff, u_ff, SAME, "grad_face_features")
    del u_feat, u_idx, u_soft, u_fvi, u_ff

    p_fvi, p_ff = t_fvi.clone().requires_grad_(True), ff16.clone().requires_grad_(True)
    p_feat, p_soft, p_idx = dibr_rasterization(H, W, t_fvz, p_fvi, p_ff, t_fnz)
    assert torch.equal(p_feat, feat) and torch.equal(p_soft, soft) and torch.equal(p_idx, idx)
    torch.autograd.backward([p_feat, p_soft], [g16, g_soft])
    assert_grad_close(p_fvi.grad, g_fvi, SAME, "public grad_face_vertices_image")
    assert_bf16_rounding_of(p_ff.grad, g_ff, "public grad_face_features")
    del p_feat, p_soft, p_idx, p_fvi, p_ff

    # the rasterize branch of views 0-1 against the oracle, on the forward's stored weights
    _, w_idx, wts, _, ws = forward_with_weights(H, W, t_fvz, t_fvi, ff16, t_fnz)
    assert torch.equal(w_idx, idx)
    r_fvi, r_ff = _host.backward(H, W, g16, None, idx, None, None, t_fvi, ff16, MULT, EPS, SIGMAINV, BOXLEN_M,
                                 KNUM, ws, True)
    o_gxy, o_gff = oracle.rasterize_backward(npy(g16[:2]), idx[:2].cpu().numpy(), npy(wts[:2]), fvi[:2],
                                             npy(ff16[:2]))
    assert_grad_close(r_fvi[:2], o_gxy, TOL, "grad_face_vertices_image, views 0-1")
    assert_grad_close(r_ff[:2], o_gff, TOL, "grad_face_features, views 0-1")


# ---------------------------------------------------------------------------------------------------
# inputs at a one-element storage offset
ALIGN_H, ALIGN_W = 96, 128


def offset(x):
    """The same values as a contiguous view one element into a larger buffer (not 16-byte aligned)."""
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device=x.device)
    buf[1:].copy_(x.reshape(-1))
    v = buf[1:].view(x.shape)
    assert v.is_contiguous() and v.data_ptr() % 16 != 0
    return v


def align_inputs(ft):
    fvz, fvi, fnz = synthetic.icosphere_views(2, 3, seed=61)
    B, F = fvz.shape[:2]
    dt = BF16 if ft == "bf16" else torch.float32
    gen = torch.Generator(device=DEV)
    gen.manual_seed(62)
    return dict(fvz=t(fvz), fvi=t(fvi), fnz=t(fnz), ff=t(synthetic.random_features(B, F, 3, seed=63)).to(dt),
                grad_features=torch.rand((B, ALIGN_H, ALIGN_W, 3), device=DEV, generator=gen).to(dt),
                grad_soft_mask=torch.rand((B, ALIGN_H, ALIGN_W), device=DEV, generator=gen))


@pytest.mark.parametrize("ft", ["fp32", "bf16"])
@pytest.mark.parametrize("which", ["fvz", "fvi", "ff", "fnz", "grad_features", "grad_soft_mask"])
def test_fused_input_at_an_element_offset(which, ft):
    """_host.forward / _host.backward copy an input that does not start on a 16-byte boundary."""
    H, W = ALIGN_H, ALIGN_W

    def fused(x):
        feat, idx, _, soft, ws = _host.forward(_lib.RASTER | _lib.SOFT_MASK, H, W, x["fvz"], x["fvi"], x["ff"],
                                               x["fnz"], None, MULT, EPS, SIGMAINV, BOXLEN_M, KNUM)
        (g_fvi, g_ff), ran = traced(_host.backward, H, W, x["grad_features"], x["grad_soft_mask"], idx, None, soft,
                                    x["fvi"], x["ff"], MULT, EPS, SIGMAINV, BOXLEN_M, KNUM, ws, True)
        assert ROWS in ran, ran
        return feat, idx, soft, g_fvi, g_ff

    x = align_inputs(ft)
    ref = fused(x)
    assert (ref[1] >= 0).any()
    x[which] = offset(x[which])
    got = fused(x)
    for a, b, what in zip(got[:3], ref[:3], ("features", "face_idx", "soft_mask")):
        assert torch.equal(a, b), what
    assert_grad_close(got[3], ref[3], SAME, "grad_face_vertices_image")
    assert_grad_close(got[4], ref[4], SAME, "grad_face_features")


@pytest.mark.parametrize("ft", ["fp32", "bf16"])
def test_public_api_at_an_element_offset(ft):
    """dibr_rasterization, rasterize and dibr_soft_mask (with a user-supplied selected_face_idx) serve
    every input at a one-element offset with the aligned call's results."""
    H, W = ALIGN_H, ALIGN_W
    x = align_inputs(ft)

    def run(move):
        m = (lambda v: offset(v)) if move else (lambda v: v.clone())
        fvi, ff = m(x["fvi"]).requires_grad_(True), m(x["ff"]).requires_grad_(True)
        feat, soft, idx = dibr_rasterization(H, W, m(x["fvz"]), fvi, ff, m(x["fnz"]))
        torch.autograd.backward([feat, soft], [m(x["grad_features"]), m(x["grad_soft_mask"])])
        r_fvi = m(x["fvi"]).requires_grad_(True)
        r_feat, r_idx = rasterize(H, W, m(x["fvz"]), r_fvi, m(x["ff"]), valid_faces=m(x["fnz"]) >= 0)
        r_feat.backward(m(x["grad_features"]))
        s_fvi = m(x["fvi"]).requires_grad_(True)
        s_soft = dibr_soft_mask(s_fvi, m(idx))
        s_soft.backward(m(x["grad_soft_mask"]))
        return (feat, soft, idx, r_feat, r_idx, s_soft), (fvi.grad, ff.grad, r_fvi.grad, s_fvi.grad)

    ref_out, ref_grads = run(False)
    got_out, got_grads = run(True)
    for a, b in zip(got_out, ref_out):
        assert torch.equal(a, b)
    for a, b in zip(got_grads, ref_grads):
        assert_grad_close(a, b, SAME, "gradient")


def test_operator_backward_at_an_element_offset():
    """The operator-contract rasterize backward runs through dibr_b200_backward, so its shim copies a
    misaligned input the same way."""
    from kaolin_b200 import _C
    x = align_inputs("fp32")
    feat, idx, wts, _, _ = forward_with_weights(ALIGN_H, ALIGN_W, x["fvz"], x["fvi"], x["ff"], x["fnz"])
    op = _C.render.mesh.rasterize_backward_cuda
    ref = op(x["grad_features"], feat, idx, wts, x["fvi"], x["ff"], EPS)
    got = op(offset(x["grad_features"]), feat, offset(idx), offset(wts), offset(x["fvi"]), offset(x["ff"]), EPS)
    for a, b, what in zip(got, ref, ("grad_face_vertices_image", "grad_face_features")):
        assert_grad_close(a, b, SAME, what)


def test_misaligned_out_buffer_raises():
    x = align_inputs("fp32")
    H, W = ALIGN_H, ALIGN_W
    _, idx, _, soft, ws = _host.forward(_lib.RASTER | _lib.SOFT_MASK, H, W, x["fvz"], x["fvi"], x["ff"], x["fnz"],
                                        None, MULT, EPS, SIGMAINV, BOXLEN_M, KNUM)
    g_fvi, g_ff = offset(torch.zeros_like(x["fvi"])), torch.zeros(x["ff"].shape, device=DEV)
    with pytest.raises(ValueError, match="16-byte"):
        _host.backward(H, W, x["grad_features"], x["grad_soft_mask"], idx, None, soft, x["fvi"], x["ff"], MULT, EPS,
                       SIGMAINV, BOXLEN_M, KNUM, ws, True, views=(0, 2), out=(g_fvi, g_ff))
