"""Argument errors are reported before any work is enqueued.

The fused backward entry points (dibr_b200_backward, _bf16, _views, _f64) get correctly sized device
buffers with one argument wrong at a time (including a tensor pointer that is not 16-byte aligned); the gradient outputs
hold a NaN sentinel.  A rejected call
returns its error code, launches no kernel (the per-kernel trace is empty) and leaves the outputs as
they were (checked after a synchronise, so a memset would show too).  The same buffers with every
argument right run the backward and overwrite the sentinel.

The float64 public wrappers apply the float32 wrappers' device and shape checks, so malformed inputs
raise before a launch.  And the float64 dibr_rasterization runs through the same autograd node as
float32, which multi_gpu's attach() finds and hooks.
"""
import pytest
import torch

from kaolin_b200 import _lib, multi_gpu, synthetic
from kaolin_b200.render.mesh import _host, dibr_rasterization, dibr_soft_mask, rasterize

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
H, W, D = 32, 48, 3
MULT, EPS, SIGMAINV, BOXLEN_M, KNUM = 1000., 1e-8, 7000., 20., 30


def _scene(dtype):
    fvz, fvi, fnz = synthetic.icosphere_views(2, 1, seed=11)
    t = lambda a: torch.from_numpy(a).to(DEV, dtype)
    return t(fvz), t(fvi), t(fnz), t(synthetic.random_features(2, fvz.shape[1], D, seed=12))


def _backward_args(entry):
    """Keyword arguments of a valid call of ``entry`` after a forward of the same scene."""
    dt = torch.float64 if entry == "f64" else torch.float32
    fvz, fvi, fnz, ff = _scene(dt)
    _, idx, wts, soft, _ = _host.forward(3, H, W, fvz, fvi, ff, fnz, None, MULT, EPS, SIGMAINV, BOXLEN_M, KNUM)
    if entry == "bf16":
        ff = ff.to(torch.bfloat16)
    gen = torch.Generator(device=DEV); gen.manual_seed(13)
    B, F = fvi.shape[:2]
    return dict(B=B, F=F, g_feat=torch.rand((B, H, W, D), device=DEV, generator=gen, dtype=dt).to(ff.dtype),
                g_soft=torch.rand((B, H, W), device=DEV, generator=gen, dtype=dt), idx=idx, wts=wts, soft=soft,
                fvi=fvi, ff=ff, mult=MULT, knum=KNUM, g_fvi=torch.empty_like(fvi),
                g_ff=torch.empty(ff.shape, dtype=dt, device=DEV),
                ws=_host.workspace(B, B * F, H, W, DEV, f64=entry == "f64"))


def _call(entry, a):
    p = _host.ptr
    ws_bytes = a["ws"].numel()
    head = (a["B"], a["F"], H, W, D, p(a["g_feat"]), p(a["g_soft"]), p(a["idx"]), p(a["wts"]), p(a["soft"]),
            p(a["fvi"]), p(a["ff"]))
    lib = _lib.lib()
    if entry == "views":
        return lib.dibr_b200_backward_views(*head, 0, a["mult"], EPS, SIGMAINV, BOXLEN_M, a["knum"], p(a["g_fvi"]),
                                            p(a["g_ff"]), p(a["ws"]), ws_bytes, 0, 1, 2, _host.stream_ptr(DEV))
    fn = {"fp32": lib.dibr_b200_backward, "bf16": lib.dibr_b200_backward_bf16, "f64": lib.dibr_b200_backward_f64}
    return fn[entry](*head, a["mult"], EPS, SIGMAINV, BOXLEN_M, a["knum"], p(a["g_fvi"]), p(a["g_ff"]), p(a["ws"]),
                     ws_bytes, 0, _host.stream_ptr(DEV))


def _traced_call(entry, a, outputs):
    """-> (status, names of the kernels launched); ``outputs`` are filled with NaN first."""
    for t in outputs:
        t.fill_(float("nan"))
    torch.cuda.synchronize()
    _lib.trace_begin()
    st = _call(entry, a)
    ran = [name for name, _ in _lib.trace_end()]
    torch.cuda.synchronize()
    return st, ran


ENTRIES = ["fp32", "bf16", "views", "f64"]


@pytest.mark.parametrize("entry", ENTRIES)
def test_valid_backward_runs(entry):
    a = _backward_args(entry)
    st, ran = _traced_call(entry, a, (a["g_fvi"], a["g_ff"]))
    assert st == 0 and ran, (st, ran)
    rows = slice(1, 2) if entry == "views" else slice(None)
    assert not torch.isnan(a["g_fvi"][rows]).any() and not torch.isnan(a["g_ff"][rows]).any()


REJECTED = [  # (id, the one wrong argument, expected status)
    ("soft_mask_null", dict(soft=None), _lib.EINVAL),
    ("knum_zero", dict(knum=0), _lib.EINVAL),
    ("workspace_one_byte_short", dict(ws="short"), _lib.EWORKSPACE),
    ("face_features_null", dict(ff=None), _lib.EINVAL),
    ("grad_face_features_null", dict(g_ff=None), _lib.EINVAL),
    ("multiplier_zero", dict(mult=0.), _lib.EINVAL),
    ("grad_features_misaligned", dict(g_feat="offset"), _lib.EINVAL),
]


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("case", REJECTED, ids=[c[0] for c in REJECTED])
def test_rejected_backward_enqueues_nothing(entry, case):
    _, wrong, code = case
    a = _backward_args(entry)
    outputs = (a["g_fvi"], a["g_ff"])
    if wrong.get("ws") == "short":      # a real allocation one byte smaller than the minimum
        wrong = dict(ws=torch.empty(a["ws"].numel() - 1, dtype=torch.uint8, device=DEV))
    if wrong.get("g_feat") == "offset":  # the same values one element into a valid buffer
        g = a["g_feat"]
        buf = torch.empty(g.numel() + 1, dtype=g.dtype, device=DEV)
        buf[1:].copy_(g.reshape(-1))
        wrong = dict(g_feat=buf[1:].view(g.shape))
        assert wrong["g_feat"].data_ptr() % 16 != 0
    a.update(wrong)
    st, ran = _traced_call(entry, a, outputs)
    assert st == code, st
    assert ran == []
    assert all(torch.isnan(t).all() for t in outputs)


def test_rejected_float64_backward_without_weights():
    a = _backward_args("f64")
    a["wts"] = None
    outputs = (a["g_fvi"], a["g_ff"])
    st, ran = _traced_call("f64", a, outputs)
    assert st == _lib.EINVAL and ran == []
    assert all(torch.isnan(t).all() for t in outputs)


def _raises_before_launch(fn, match):
    _lib.trace_begin()
    try:
        with pytest.raises(RuntimeError, match=match):
            fn()
    finally:
        ran = [name for name, _ in _lib.trace_end()]
    assert ran == []


def test_float64_soft_mask_checks_its_inputs():
    fvz, fvi, fnz, ff = _scene(torch.float64)
    _, idx = rasterize(H, W, fvz, fvi, ff)
    assert idx.dtype == torch.int64
    assert dibr_soft_mask(fvi, idx).dtype == torch.float64
    _raises_before_launch(lambda: dibr_soft_mask(fvi, idx.int()), "LongTensor")
    _raises_before_launch(lambda: dibr_soft_mask(fvi, torch.cat([idx, idx])), "LongTensor")
    _raises_before_launch(lambda: dibr_soft_mask(fvi[:, :, :2].contiguous(), idx), r"\(batch_size, num_faces, 3, 2\)")


def test_float64_rasterize_checks_valid_faces():
    fvz, fvi, fnz, ff = _scene(torch.float64)
    B, F = fvz.shape[:2]
    valid = fnz >= 0
    _raises_before_launch(lambda: rasterize(H, W, fvz, fvi, ff, valid_faces=valid[:, :F - 1]), "valid_faces")
    _raises_before_launch(lambda: rasterize(H, W, fvz, fvi, ff, valid_faces=valid.cpu()), "CUDA")


def test_float64_backward_rejects_view_chunks():
    a = _backward_args("f64")
    with pytest.raises(ValueError):
        _host.backward(H, W, a["g_feat"], a["g_soft"], a["idx"], a["wts"], a["soft"], a["fvi"], a["ff"], MULT, EPS,
                       SIGMAINV, BOXLEN_M, KNUM, None, False, views=(0, 1))


def test_attach_finds_the_float64_dibr_node_through_a_slice():
    """attach() finds the node of a float64 dibr_rasterization call (through a slice of a list/tuple
    feature output); the float64 backward, one kernel, calls the hook once at its end with the final
    float64 feature gradient, and runs in one piece even with a view pipeline attached."""
    fvz, fvi, fnz, ff = _scene(torch.float64)
    t_fvi, t_ff = fvi.clone().requires_grad_(True), ff.clone().requires_grad_(True)
    (fa, fb), soft, _ = dibr_rasterization(H, W, fvz, t_fvi, [t_ff[..., :2], t_ff[..., 2:]], fnz)
    node = multi_gpu._dibr_node(fa)
    assert node is multi_gpu._dibr_node(soft) and type(node).__name__.startswith("DibrRasterizationB200")
    hooked = []
    g = object.__new__(multi_gpu.OverlappedGradAllGather)      # no process group needed for attach()
    g.hook = lambda t: hooked.append(t.clone())
    assert g.attach(fb) is g and node.feature_grad_hook is g.hook
    node.view_pipeline = lambda *args: pytest.fail("the float64 backward does not run in view chunks")
    gen = torch.Generator(device=DEV); gen.manual_seed(14)
    grads = [torch.rand(x.shape, device=DEV, generator=gen, dtype=torch.float64) for x in (fa, fb, soft)]
    torch.autograd.backward([fa, fb, soft], grads)
    assert len(hooked) == 1
    assert hooked[0].dtype == torch.float64 and torch.equal(hooked[0], t_ff.grad)
