"""sg_shade on its fused sm_90a kernels: against the reference's goldens (tests/golden/shade.npz),
against the fp64 restatement (oracle/shade.py) on a batch of views, against the reference's
structure composed from this library's two lighting calls, and for exact background zeros,
bit-reproducible light gradients, sync-free calls and edge sizes.  Tolerance 1e-5 of the tensor's
scale."""
import math
import os
import types

import numpy as np
import pytest
import torch

from oracle import shade as OSH
from kaolin_b200 import _lib
from kaolin_b200.render import easy_render, lighting

pytestmark = pytest.mark.gpu
DEV = "cuda"
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "shade.npz"))
NAMES = ("albedo", "spec_albedo", "roughness", "normals", "amp", "dir", "sharp")
OUTS = ("diffuse", "specular", "img")


class Cam(types.SimpleNamespace):
    def __len__(self):
        return self.extrinsics.R.shape[0]


def golden_camera(B=1):
    t = lambda k: torch.from_numpy(G[k]).float().to(DEV).repeat(*([B] + [1] * (G[k].ndim - 1)))
    return Cam(extrinsics=types.SimpleNamespace(R=t("cam_R")), x0=t("cam_x0"), y0=t("cam_y0"),
               focal_x=t("cam_focal_x"), focal_y=t("cam_focal_y"), width=int(G["cam_width"]),
               height=int(G["cam_height"]))


def err(a, ref):
    a, ref = a.detach().double().cpu(), ref.detach().double().cpu()
    assert a.shape == ref.shape, (a.shape, ref.shape)
    if ref.numel() == 0:
        return 0.0
    return float((a - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)


def close(a, ref, tol=1e-5):
    e = err(a, ref)
    assert e <= tol, e
    return e


def golden_inputs(L):
    face_idx = torch.from_numpy(G[f"L{L}_face_idx"]).to(DEV)
    return face_idx, [torch.from_numpy(G[f"L{L}_{k}"]).float().to(DEV) for k in NAMES]


def run(fn, cam, face_idx, ins, ws):
    leaves = [t.detach().clone().requires_grad_(True) for t in ins]
    outs = fn(cam, face_idx, *leaves)
    sum((o * w).sum() for o, w in zip(outs, ws) if w is not None).backward()
    return outs, [t.grad for t in leaves]


def composed(cam, face_idx, albedo, spec_albedo, roughness, normals, amp, dirs, sharp):
    """The reference's sg_shade structure on this library's two lighting calls."""
    mask = face_idx >= 0
    n = torch.nn.functional.normalize(normals[mask], dim=-1)
    d = lighting.sg_diffuse_inner_product(amp, dirs, sharp, n, albedo[mask])
    view = OSH.view_dirs(cam.extrinsics.R.double().cpu(), cam.x0.double().cpu(), cam.y0.double().cpu(),
                         cam.focal_x.double().cpu(), cam.focal_y.double().cpu(), cam.width, cam.height,
                         *face_idx.shape[1:]).float().to(DEV)
    s = lighting.sg_warp_specular_term(amp, dirs, sharp, n, roughness[mask].reshape(-1), view[mask].contiguous(),
                                       spec_albedo[mask])
    z = torch.zeros(face_idx.shape + (3,), device=DEV)
    return z.index_put((mask,), d), z.index_put((mask,), s), z.index_put((mask,), d + s)


@pytest.mark.parametrize("L", (1, 2, 7, 8, 40))
def test_goldens(L):
    face_idx, ins = golden_inputs(L)
    ws = [torch.from_numpy(G[f"L{L}_w_{n}"]).float().to(DEV) for n in OUTS]
    outs, grads = run(easy_render.sg_shade, golden_camera(), face_idx, ins, ws)
    for o, n in zip(outs, OUTS):
        close(o, torch.from_numpy(G[f"L{L}_{n}"]))
    for gr, k in zip(grads, NAMES):
        close(gr, torch.from_numpy(G[f"L{L}_g_{k}"]))


def batch(B, H, W, L, seed, coverage=0.7):
    """B views of the golden camera's pose: normals with n.v in [0.25, 1] of each pixel's view, the
    value ranges of texture_sample_materials, roughness in [0.3, 1]."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    cam = golden_camera(B)
    view = OSH.view_dirs(cam.extrinsics.R.double().cpu(), cam.x0.double().cpu(), cam.y0.double().cpu(),
                         cam.focal_x.double().cpu(), cam.focal_y.double().cpu(), cam.width, cam.height, H, W).to(DEV)
    rnd = lambda *s: torch.rand(s, device=DEV, generator=gen, dtype=torch.float64)
    face_idx = torch.where(rnd(B, H, W) < coverage, (rnd(B, H, W) * 1000).long(), -1)
    face_idx[:, : H // 4] = -1                                      # whole background rows
    t = torch.nn.functional.normalize(torch.randn((B, H, W, 3), device=DEV, generator=gen, dtype=torch.float64), dim=-1)
    t = torch.nn.functional.normalize(t - (t * view).sum(-1, keepdim=True) * view, dim=-1)
    c = 0.25 + 0.75 * rnd(B, H, W, 1)
    normals = (c * view + torch.sqrt(1 - c * c) * t) * (0.8 + 0.4 * rnd(B, H, W, 1))
    base, metal = rnd(B, H, W, 3), rnd(B, H, W, 1)
    amp = rnd(L, 3) * 2
    dirs = torch.nn.functional.normalize(torch.randn((L, 3), device=DEV, generator=gen, dtype=torch.float64), dim=-1)
    sharp = torch.exp(rnd(L) * math.log(100.)) * 0.5
    ins = [base * (1 - metal), (1 - metal) * 0.04 + base * metal, 0.3 + 0.7 * rnd(B, H, W, 1), normals, amp, dirs, sharp]
    ws = [rnd(B, H, W, 3) - 0.3 for _ in range(3)]
    return cam, face_idx, [x.float() for x in ins], [w.float() for w in ws]


def kinks(view, normals, tol=1e-4):
    """(B,H,W): pixels where fp32 may take the other side of a specular clamp than fp64: n.v at 1,
    n.w (w the warped lobe direction) or l.h at 0 or 1."""
    n = torch.nn.functional.normalize(normals.double(), dim=-1)
    v = view.double()
    nv = (n * v).sum(-1, keepdim=True)
    w = -v + 2 * nv * n
    h = w + v
    h = h / h.norm(dim=-1, keepdim=True)
    near = torch.zeros(nv.shape[:-1], dtype=torch.bool, device=nv.device)
    for x in (nv[..., 0], (n * w).sum(-1), (w * h).sum(-1)):
        near |= ((x.abs() < tol) | ((x - 1).abs() < tol))
    return near


@pytest.mark.parametrize("L", (1, 8, 32, 129))
def test_against_the_fp64_oracle(L):
    cam, face_idx, ins, ws = batch(8, 96, 136, L, seed=L)
    outs, grads = run(easy_render.sg_shade, cam, face_idx, ins, ws)
    view = OSH.view_dirs(cam.extrinsics.R.double().cpu(), cam.x0.double().cpu(), cam.y0.double().cpu(),
                         cam.focal_x.double().cpu(), cam.focal_y.double().cpu(), cam.width, cam.height, 96, 136)
    o64, g64 = run(lambda c, f, *a: OSH.sg_shade(view.to(DEV), f, *a), cam, face_idx,
                   [x.double() for x in ins], [w.double() for w in ws])
    o32, g32 = run(lambda c, f, *a: OSH.sg_shade(view.to(DEV).float(), f, *a), cam, face_idx, ins, ws)
    for o, r in zip(outs, o64):
        close(o, r)
    away = ~kinks(view.to(DEV), ins[3])
    assert away.float().mean() > 0.99
    for i, (k, gr, r, r32) in enumerate(zip(NAMES, grads, g64, g32)):
        if i < 4:                                                     # per-pixel gradients: away from the kinks
            gr, r, r32 = gr[away], r[away], r32[away]
        # the roughness gradient's lobe terms nearly cancel in fp32 (DESIGN.md, f6): 4x the fp32 formula's error
        close(gr, r, max(1e-5, 4 * err(r32, r)) if k == "roughness" else 1e-5)


@pytest.mark.parametrize("which", (0, 1, 2, None))
def test_equals_the_composed_path(which):
    cam, face_idx, ins, ws = batch(3, 40, 52, 9, seed=7)
    ws = [w if which in (None, i) else None for i, w in enumerate(ws)]
    outs, grads = run(easy_render.sg_shade, cam, face_idx, ins, ws)
    ro, rg = run(composed, cam, face_idx, ins, ws)
    for o, r in zip(outs, ro):
        close(o, r)
    for gr, r, x in zip(grads, rg, ins):
        close(gr, torch.zeros_like(x) if r is None else r)       # no path from the loss: zero, not None


def test_distinct_cameras_per_view():
    """Every view its own pose, principal point and focal lengths; 17 x 23 pixels, so that threads'
    pixels cross view boundaries."""
    B, H, W = 3, 17, 23
    cam, face_idx, ins, ws = batch(B, H, W, 6, seed=19, coverage=0.9)
    ang = torch.tensor([0.0, 0.7, -1.9])
    c, s_ = torch.cos(ang), torch.sin(ang)
    Ry = torch.stack([torch.stack([c, torch.zeros(3), s_], -1), torch.tensor([[0., 1., 0.]]).expand(3, 3),
                      torch.stack([-s_, torch.zeros(3), c], -1)], 1)            # (B, 3, 3) rotations about y
    cam.extrinsics.R = (Ry @ cam.extrinsics.R.cpu()).to(DEV)
    cam.x0 = torch.tensor([7.5, -12.0, 0.25], device=DEV)
    cam.y0 = torch.tensor([-4.25, 9.5, 3.0], device=DEV)
    cam.focal_x = cam.focal_x * torch.tensor([1.0, 0.8, 1.3], device=DEV)
    cam.focal_y = cam.focal_y * torch.tensor([1.1, 0.7, 1.2], device=DEV)
    views = OSH.view_dirs(cam.extrinsics.R.double().cpu(), cam.x0.double().cpu(), cam.y0.double().cpu(),
                          cam.focal_x.double().cpu(), cam.focal_y.double().cpu(), cam.width, cam.height, H, W)
    assert (views[0] - views[1]).abs().max() > 0.1 and (views[1] - views[2]).abs().max() > 0.1
    # normals facing each view's own rays, so the specular term is well conditioned in every view
    n = torch.nn.functional.normalize(views.to(DEV).float() + 0.3 * torch.nn.functional.normalize(ins[3], dim=-1), dim=-1)
    ins[3] = n * ins[3].norm(dim=-1, keepdim=True)
    outs, grads = run(easy_render.sg_shade, cam, face_idx, ins, ws)
    ro, rg = run(composed, cam, face_idx, ins, ws)
    for o, r in zip(outs, ro):
        close(o, r)
    for gr, r in zip(grads, rg):
        close(gr, r)
    o64, _ = run(lambda c, f, *a: OSH.sg_shade(views.to(DEV), f, *a), cam, face_idx, [x.double() for x in ins],
                 [w.double() for w in ws])
    for o, r in zip(outs, o64):
        close(o, r)


def test_background_is_exactly_zero():
    cam, face_idx, ins, ws = batch(2, 33, 47, 5, seed=3)
    ins[3] = ins[3].clone()
    ins[3][face_idx < 0] = float("nan")                               # background values are never read
    ins[2] = ins[2].clone()
    ins[2][face_idx < 0] = 0.
    outs, grads = run(easy_render.sg_shade, cam, face_idx, ins, ws)
    bg = face_idx < 0
    for o in outs:
        assert (o[bg] == 0).all()
        assert torch.isfinite(o).all()
    for gr in grads[:4]:
        assert (gr[bg] == 0).all()
    for gr in grads[4:]:
        assert torch.isfinite(gr).all()


def test_light_gradients_are_reproducible_and_independent_of_the_per_pixel_ones():
    cam, face_idx, ins, ws = batch(4, 64, 80, 70, seed=11)
    _, g1 = run(easy_render.sg_shade, cam, face_idx, ins, ws)
    _, g2 = run(easy_render.sg_shade, cam, face_idx, ins, ws)
    lights = [t.detach().clone().requires_grad_(True) for t in ins[4:]]
    outs = easy_render.sg_shade(cam, face_idx, *ins[:4], *lights)
    sum((o * w).sum() for o, w in zip(outs, ws)).backward()
    for a, b, c in zip(g1[4:], g2[4:], lights):
        assert torch.equal(a, b)
        assert torch.equal(a, c.grad)


def test_no_host_synchronisation():
    cam, face_idx, ins, ws = batch(2, 32, 40, 3, seed=5)
    leaves = [t.detach().clone().requires_grad_(True) for t in ins]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        outs = easy_render.sg_shade(cam, face_idx, *leaves)
        torch.autograd.backward(outs, ws)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


@pytest.mark.parametrize("B,H,W,L,cov", [(2, 17, 23, 0, 0.7), (2, 17, 23, 3, 0.0), (1, 1, 1, 2, 1.0),
                                         (3, 31, 29, 65, 0.8), (1, 7, 300, 4, 0.9)])
def test_edge_sizes(B, H, W, L, cov):
    cam, face_idx, ins, ws = batch(B, H, W, L, seed=H * W + L, coverage=cov)
    if H == 1:
        face_idx[:] = 0
    outs, grads = run(easy_render.sg_shade, cam, face_idx, ins, ws)
    ro, rg = run(composed, cam, face_idx, ins, ws)
    for o, r in zip(outs, ro):
        close(o, r)
    for gr, r in zip(grads, rg):
        close(gr, r)


def test_workspace_at_an_odd_address(monkeypatch):
    """Every workspace starting at byte 1 of a larger buffer: the outputs of an aligned one."""
    cam, face_idx, ins, ws = batch(2, 32, 40, 5, seed=13)

    def shade():
        outs, grads = run(easy_render.sg_shade, cam, face_idx, ins, ws)
        return [*outs, *grads]

    want = shade()
    scratch, odd = _lib.scratch, []
    monkeypatch.setattr(_lib, "scratch", lambda n, device: odd.append(n) or scratch(int(n) + 1, device)[1:])
    got = shade()
    assert odd
    for a, b in zip(want, got):
        assert torch.equal(a, b)
