"""The judge of tests/test_pipeline_edges_gpu.py is oracle/pipeline.py's torch restatements run in
float64.  Here they are pinned to the reference's own functions run in float64 on the same edge
scenes (tests/golden/pipeline_edges.npz, written by tests/golden/make_pipeline_edges_golden.py):
zero-area faces, the scale where the normal's 1e-10 matters, every pair of clamp / border kink
coordinates, and empty / full / out-of-range masks.  1e-12, relative to each element."""
import os

import numpy as np
import pytest
import torch

from oracle import pipeline as P

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "pipeline_edges.npz"))
D = torch.float64
T = lambda k, grad=False: torch.from_numpy(G[k]).to(D).requires_grad_(grad)


def same(a, key, tol=1e-12, largest=None):
    a, ref = a.detach().numpy(), G[key]
    assert a.shape == ref.shape and a.dtype == ref.dtype == np.float64, key
    assert np.array_equal(np.isnan(a), np.isnan(ref)), key
    # a zero-area face sends +-1e10-sized terms (g_n / 1e-10) to its vertices, which cancel there: the
    # sum carries float64 rounding of its largest term, hence the second part (`largest`: the size of
    # that term where the tensor itself, a camera gradient summed over the vertices, no longer shows it)
    largest = np.nanmax(np.abs(ref), initial=0) if largest is None else largest
    ok = np.abs(a - ref) <= tol * (1 + np.abs(ref)) + 8 * 2.0 ** -53 * largest
    assert np.all(ok | np.isnan(ref)), (key, float(np.nanmax(np.abs(a - ref))))


@pytest.mark.parametrize("mode", ["T", "Rt"])
@pytest.mark.parametrize("tag", ["dg", "ep"])
def test_prepare_vertices_float64_restatement(tag, mode):
    v = T(f"{tag}_vertices", True)
    if mode == "T":
        cam = dict(camera_transform=T(f"{tag}_transform", True))
    else:
        cam = dict(camera_rot=T(f"{tag}_rot", True), camera_trans=T(f"{tag}_trans", True))
    res = P.prepare_vertices_torch(v, torch.from_numpy(G[f"{tag}_faces"]), T(f"{tag}_proj"), **cam)
    sum((o * T(f"{tag}_w{i + 1}")).sum() for i, o in enumerate(res)).backward()
    for name, o in zip(("fvc", "fvi", "fn"), res):
        same(o, f"{tag}_{mode}_{name}")
    same(v.grad, f"{tag}_{mode}_g_vertices")
    for name, t in cam.items():
        same(t.grad, f"{tag}_{mode}_g_{name[7:]}", largest=np.abs(G[f"{tag}_{mode}_g_vertices"]).max())


def test_golden_scenes_do_their_job():
    """The scenes keep the properties the GPU tests rely on."""
    fn = G["dg_T_fn"]
    deg = G["dg_degenerate"]
    assert np.all(fn[:, deg] == 0) and np.all(np.abs(np.linalg.norm(np.delete(fn, deg, 1), axis=-1) - 1) < 1e-8)
    assert np.all(np.isfinite(G["dg_T_g_vertices"])) and np.all(np.isfinite(G["dg_Rt_g_vertices"]))
    fvc = G["ep_T_fvc"]
    L = np.linalg.norm(np.cross(fvc[:, :, 1] - fvc[:, :, 0], fvc[:, :, 2] - fvc[:, :, 0]), axis=-1)
    assert L.min() < 1e-13 and L.max() > 1e-7 and ((L > 1e-11) & (L < 1e-9)).any()
    # un-normalised: with 1e-10 in the denominator the "unit" normals of the small views are not unit
    n = np.linalg.norm(G["ep_T_fn"], axis=-1)
    assert n.min() < 0.01 and n.max() > 0.999


@pytest.mark.parametrize("mode", ["nearest", "bilinear"])
@pytest.mark.parametrize("tag", ["tk51", "tk48"])
def test_texture_mapping_float64_restatement(tag, mode):
    uv, tex = T(f"{tag}_uv", True), T(f"{tag}_tex", True)
    o = P.texture_mapping_torch(uv, tex, mode=mode)
    (o * T(f"{tag}_gw")).sum().backward()
    same(o, f"{tag}_{mode}_out"); same(tex.grad, f"{tag}_{mode}_g_tex")
    same(uv.grad if uv.grad is not None else torch.zeros_like(uv), f"{tag}_{mode}_g_uv")
    if mode == "bilinear":       # the grid holds both sides of every kink
        g = G[f"{tag}_bilinear_g_uv"]
        assert (g[..., 1] != 0).any() and (g == 0).any() and (tag == "tk51" or (g[..., 0] != 0).any())


@pytest.mark.parametrize("name", ["empty", "full", "one_empty", "complement", "range"])
def test_mask_iou_float64_restatement(name):
    l, r = T(f"mi_{name}_lhs", True), T(f"mi_{name}_rhs", True)
    loss = P.mask_iou_torch(l, r)
    (loss * float(G["mi_gscale"])).backward()
    assert abs(loss.item() - float(G[f"mi_{name}_loss"])) <= 1e-12
    same(l.grad, f"mi_{name}_g_lhs"); same(r.grad, f"mi_{name}_g_rhs")
    if name == "empty":
        assert loss.item() == 1.0 and not l.grad.any() and not r.grad.any()
