"""Regenerates tests/golden/shade.npz and tests/golden/render_mesh.npz from the reference (run where its
sources are present).

    python tests/golden/make_shade_golden.py

Outputs and autograd gradients of the reference's OWN kaolin.render.easy_render.mesh.sg_shade
(mesh.py:427-464), imported in place, on a float64 Camera and float64 G-buffers: the three images and
the gradients of albedo, spec_albedo, roughness, normals and the lights under a random weighting of
all three outputs.  The reference allocates its images as ``torch.float``; the module's ``torch`` is
given a view of torch whose ``float`` is float64, so that the function runs unchanged in float64.
Under the stub ``_C`` the
reference's fused inner-product operator returns None for 8 or more lights, so for those sizes the
lighting module's ``unbatched_reduced_sg_inner_product`` is rebound to the reference's own composition,
``unbatched_sg_inner_product(...).sum(1)``, as in make_specular_golden.py.

shade.npz: the camera (stored as plain arrays) has a non-zero principal point offset (x0, y0), a 320 x 240 image,
and the G-buffer is 24 x 20, so the ray grid is the custom-resolution one.  A quarter of the pixels are
background; normals are of norm 0.8-1.2 with n.v in [0.25, 1] (a few face away from the view); albedo
and spec_albedo are in the ranges the metallic-roughness workflow of texture_sample_materials gives
(spec_albedo in [0.04, 1]); roughness is in [0.3, 1].

render_mesh.npz: the reference's render_mesh(backend='cuda') in float32, its rasterizer operator played
by the oracle's restatement (oracle.packed_rasterize_forward), on a level-2 icosphere SurfaceMesh with
spherical uvs and two materials chosen per face by material_assignments: a metallic-roughness
PBRMaterial with diffuse, normal, roughness and metallic textures, and a specular-workflow one with
constant colours and roughness.  Once with the default light, once with three lights; in the second
run the lights and the first material's diffuse and roughness textures require grad, and their
gradients under a random weighting of the rendered image are stored.  The mesh attributes the renderer
reads, the materials and the camera's transforms of the vertices are stored as plain arrays, so that a
test can rebuild duck-typed stand-ins without the reference.
"""
import math
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))
import oracle  # noqa: E402
from oracle import ref_import  # noqa: E402
from kaolin_b200 import synthetic  # noqa: E402


def _packed_rasterize_forward(height, width, z, xy, bboxes, features, first, multiplier, eps):
    """The reference's rasterizer operator, played by the oracle's C restatement on the CPU."""
    out, idx, w = oracle.packed_rasterize_forward(height, width, *(t.detach().numpy() for t in (z, xy, bboxes, features)),
                                                  first.numpy(), multiplier, eps)
    return torch.from_numpy(out), torch.from_numpy(idx), torch.from_numpy(w)


_C = ref_import._Stub("kaolin._C")
_C.render.mesh.packed_rasterize_forward_cuda = _packed_rasterize_forward
ref_import.setup(_C)
easy = ref_import.module("kaolin.render.easy_render.mesh")
sg = ref_import.module("kaolin.render.lighting.sg")
camera_mod = ref_import.module("kaolin.render.camera")
raygen = ref_import.module("kaolin.render.camera.raygen")
_fused = sg.unbatched_reduced_sg_inner_product


class _Float64Torch:
    float = torch.float64

    def __getattr__(self, k):
        return getattr(torch, k)


easy.torch = _Float64Torch()
D = torch.float64
g = torch.Generator().manual_seed(20261017)


def unit(*shape):
    v = torch.randn(shape + (3,), generator=g, dtype=D)
    return v / v.norm(dim=-1, keepdim=True)


cam = camera_mod.Camera.from_args(eye=torch.tensor([1.3, 0.9, 2.1]), at=torch.tensor([0.1, -0.05, 0.]),
                                  up=torch.tensor([0., 1., 0.]), fov=math.pi * 40 / 180, width=320, height=240,
                                  x0=7.5, y0=-4.25, dtype=D)
H, W = 20, 24
grid = raygen.generate_centered_custom_resolution_pixel_coords(cam.width, cam.height, res_x=W, res_y=H)
_, rays_d = raygen.generate_pinhole_rays(cam, grid)
view = -rays_d.reshape(1, H, W, 3)

out = dict(cam_R=cam.extrinsics.R, cam_x0=cam.x0, cam_y0=cam.y0, cam_focal_x=cam.focal_x, cam_focal_y=cam.focal_y,
           cam_width=np.array(cam.width), cam_height=np.array(cam.height), view=view)
for L in (1, 2, 7, 8, 40):
    sg.unbatched_reduced_sg_inner_product = _fused if L < 8 else (
        lambda *a: sg.unbatched_sg_inner_product(*a).sum(1))
    face_idx = torch.randint(0, 500, (1, H, W), generator=g)
    face_idx[torch.rand((1, H, W), generator=g) < 0.25] = -1
    t = unit(1, H, W)
    t = t - (t * view).sum(-1, keepdim=True) * view
    t = t / t.norm(dim=-1, keepdim=True)
    cos = 0.25 + 0.75 * torch.rand((1, H, W, 1), generator=g, dtype=D)
    cos[0, :2, :4] = -(0.2 + 0.8 * torch.rand((2, 4, 1), generator=g, dtype=D))       # facing away
    normals = (cos * view + torch.sqrt(1 - cos * cos) * t) * (0.8 + 0.4 * torch.rand((1, H, W, 1), generator=g, dtype=D))
    base = torch.rand((1, H, W, 3), generator=g, dtype=D)
    metallic = torch.rand((1, H, W, 1), generator=g, dtype=D)
    albedo = base * (1 - metallic)
    spec_albedo = (1 - metallic) * 0.04 + base * metallic
    roughness = 0.3 + 0.7 * torch.rand((1, H, W, 1), generator=g, dtype=D)
    amp = torch.rand((L, 3), generator=g, dtype=D) * 3
    dirs = unit(L)
    sharp = torch.exp(torch.rand((L,), generator=g, dtype=D) * np.log(100.)) * 0.5
    w = [torch.rand((1, H, W, 3), generator=g, dtype=D) - 0.3 for _ in range(3)]
    ins = dict(albedo=albedo, spec_albedo=spec_albedo, roughness=roughness, normals=normals,
               amp=amp, dir=dirs, sharp=sharp)
    leaves = {k: v.clone().requires_grad_(True) for k, v in ins.items()}
    outs = easy.sg_shade(cam, face_idx, leaves["albedo"], leaves["spec_albedo"], leaves["roughness"],
                         leaves["normals"], leaves["amp"], leaves["dir"], leaves["sharp"])
    assert all(o.dtype == D for o in outs)
    sum((o * wk).sum() for o, wk in zip(outs, w)).backward()
    out[f"L{L}_face_idx"] = face_idx
    for k, v in ins.items():
        out[f"L{L}_{k}"] = v
        out[f"L{L}_g_{k}"] = leaves[k].grad
    for name, o, wk in zip(("diffuse", "specular", "img"), outs, w):
        out[f"L{L}_{name}"] = o.detach()
        out[f"L{L}_w_{name}"] = wk
    assert (outs[2][face_idx < 0] == 0).all() and (outs[1][face_idx >= 0] > 0).any(), L
sg.unbatched_reduced_sg_inner_product = _fused

out = {k: (v.detach().contiguous().numpy() if torch.is_tensor(v) else v) for k, v in out.items()}
np.savez_compressed(os.path.join(HERE, "shade.npz"), **out)
print("wrote", os.path.join(HERE, "shade.npz"), len(out), "arrays")


# ------------------------------------------------------------------------------------------------
easy.torch = torch                         # render_mesh runs in float32, as the reference does
camera_mod = ref_import.module("kaolin.render.camera")
rep = ref_import.module("kaolin.rep")
materials = ref_import.module("kaolin.render.materials")
g = torch.Generator().manual_seed(20261018)
F32 = torch.float32
v, f = synthetic.icosphere(2)
v, f = torch.from_numpy(v).to(F32), torch.from_numpy(f)
uvs = torch.stack([torch.atan2(v[:, 2], v[:, 0]) / (2 * math.pi) + 0.5, torch.acos(v[:, 1].clamp(-1, 1)) / math.pi], -1)
assignments = (v[f].mean(1)[:, 0] > 0.1).to(torch.int16)
tex = dict(diffuse_texture=torch.rand((16, 16, 3), generator=g),
           normals_texture=torch.nn.functional.normalize(
               torch.rand((16, 16, 3), generator=g) * torch.tensor([0.4, 0.4, 1.]) - torch.tensor([0.2, 0.2, 0.]), dim=-1),
           roughness_texture=0.2 + 0.8 * torch.rand((16, 16, 1), generator=g),
           metallic_texture=torch.rand((16, 16, 1), generator=g))
const = dict(diffuse_color=(0.8, 0.3, 0.2), specular_color=(0.3, 0.5, 0.7), roughness_value=0.4)
cam = camera_mod.Camera.from_args(eye=torch.tensor([2.0, 1.2, 2.4]), at=torch.zeros(3), up=torch.tensor([0., 1., 0.]),
                                  fov=math.pi * 40 / 180, width=40, height=32, x0=1.5, y0=-0.75)
vc = cam.extrinsics.transform(v)
rm = dict(vertices=v, faces=f, uvs=uvs, material_assignments=assignments, cam_R=cam.extrinsics.R, cam_x0=cam.x0,
          cam_y0=cam.y0, cam_focal_x=cam.focal_x, cam_focal_y=cam.focal_y, cam_width=np.array(cam.width),
          cam_height=np.array(cam.height), vertices_camera=vc, vertices_image=cam.intrinsics.transform(vc),
          vertices_ndc=cam.transform(v), **{f"m0_{k}": t for k, t in tex.items()},
          **{f"m1_{k}": torch.tensor(c) for k, c in const.items()})
amp = torch.rand((3, 3), generator=g) * 2
dirs = torch.nn.functional.normalize(torch.randn((3, 3), generator=g), dim=-1)
sharp = 2 + 8 * torch.rand((3,), generator=g)
w = torch.rand((1, 32, 40, 3), generator=g) - 0.3
rm.update(light_amp=amp, light_dir=dirs, light_sharp=sharp, w=w)
for run, grad in (("default", False), ("lit", True)):
    leaves = {k: t.clone().requires_grad_(grad) for k, t in tex.items()}
    mats = [materials.PBRMaterial(is_specular_workflow=False, **leaves),
            materials.PBRMaterial(is_specular_workflow=True, **const)]
    mesh = rep.SurfaceMesh(vertices=v, faces=f, uvs=uvs, face_uvs_idx=f, material_assignments=assignments,
                           materials=mats)
    lights = None
    if grad:
        lp = [t.clone().requires_grad_(True) for t in (amp, dirs, sharp)]
        lights = types.SimpleNamespace(amplitude=lp[0], direction=lp[1], sharpness=lp[2])
    res = easy.render_mesh(cam, mesh, lighting=lights, backend='cuda')
    if run == "default":
        rm.update(face_normals=mesh.face_normals, face_uvs=mesh.face_uvs, face_tangents=mesh.face_tangents)
        assert set(torch.unique(assignments[res["face_idx"][res["face_idx"] >= 0]]).tolist()) == {0, 1}
    for k, t in res.items():
        rm[f"{run}_{getattr(k, 'name', k)}"] = t
    if grad:
        (res["render"] * w).sum().backward()
        for k, t in zip(("amp", "dir", "sharp"), lp):
            rm[f"{run}_g_light_{k}"] = t.grad
        for k in ("diffuse_texture", "roughness_texture"):
            rm[f"{run}_g_m0_{k}"] = leaves[k].grad

rm = {k: (t.detach().contiguous().numpy() if torch.is_tensor(t) else t) for k, t in rm.items()}
np.savez_compressed(os.path.join(HERE, "render_mesh.npz"), **rm)
print("wrote", os.path.join(HERE, "render_mesh.npz"), len(rm), "arrays")
