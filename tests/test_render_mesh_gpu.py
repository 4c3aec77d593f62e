"""render_mesh and texture_sample_materials against the reference's own render_mesh
(tests/golden/render_mesh.npz): a textured metallic-roughness material and a constant-colour
specular-workflow one on one icosphere, chosen per face by material_assignments, under the default
light and under three lights with gradients to the lights and to two textures.  The mesh, materials
and camera are duck-typed stand-ins rebuilt from the stored arrays; the camera's transforms return
the reference camera's stored transforms of the vertices."""
import os
import types

import numpy as np
import pytest
import torch

from kaolin_b200.render import easy_render

pytestmark = pytest.mark.gpu
DEV = "cuda"
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "render_mesh.npz"))
T = lambda k: torch.from_numpy(np.ascontiguousarray(G[k])).to(DEV)


def err(a, ref):
    a, ref = a.detach().double().cpu(), ref.detach().double().cpu()
    assert a.shape == ref.shape, (a.shape, ref.shape)
    return float((a - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)


class Camera(types.SimpleNamespace):
    def __len__(self):
        return 1

    def transform(self, v):
        assert torch.equal(v, self._vertices)
        return T("vertices_ndc")


def camera(vertices):
    def ext(v):
        assert torch.equal(v, vertices)
        return T("vertices_camera")

    def intr(v):
        assert torch.equal(v, T("vertices_camera"))
        return T("vertices_image")
    return Camera(extrinsics=types.SimpleNamespace(R=T("cam_R"), transform=ext),
                  intrinsics=types.SimpleNamespace(transform=intr), x0=T("cam_x0"), y0=T("cam_y0"),
                  focal_x=T("cam_focal_x"), focal_y=T("cam_focal_y"), width=int(G["cam_width"]),
                  height=int(G["cam_height"]), dtype=torch.float32, device=torch.device(DEV), _vertices=vertices)


class Material(types.SimpleNamespace):
    TEXTURES = ("normals_texture", "diffuse_texture", "specular_texture", "metallic_texture", "roughness_texture")

    def chw(self):
        return Material(**{k: (v.permute(2, 0, 1) if k in self.TEXTURES and v is not None else v)
                           for k, v in vars(self).items()})


def materials(grad):
    tex = {k: T(f"m0_{k}").requires_grad_(grad) for k in ("diffuse_texture", "normals_texture",
                                                          "roughness_texture", "metallic_texture")}
    none = dict.fromkeys(Material.TEXTURES + ("diffuse_color", "specular_color", "metallic_value",
                                              "roughness_value"))
    m0 = Material(**{**none, **tex, "is_specular_workflow": False})
    m1 = Material(**{**none, "diffuse_color": T("m1_diffuse_color"), "specular_color": T("m1_specular_color"),
                     "roughness_value": T("m1_roughness_value"), "is_specular_workflow": True})
    return [m0, m1], tex


class Mesh(types.SimpleNamespace):
    ATTRS = ("face_normals", "face_uvs", "face_tangents")

    def __len__(self):
        return 1

    def __getitem__(self, i):
        return self

    def has_attribute(self, name):
        return name in self.ATTRS

    def has_or_can_compute_attribute(self, name):
        return name in self.ATTRS


def mesh(mats):
    return Mesh(vertices=T("vertices"), faces=T("faces"), face_normals=T("face_normals"), face_uvs=T("face_uvs"),
                face_tangents=T("face_tangents"), materials=mats, material_assignments=T("material_assignments"))


def check_passes(res, run):
    ref_keys = {k[len(run) + 1:] for k in G.files if k.startswith(run + "_") and "_g_" not in k[len(run):]}
    ref_keys = {k for k in ref_keys if not k.startswith("g_")}
    assert set(res) == ref_keys, (set(res), ref_keys)
    assert torch.equal(res["face_idx"].cpu(), torch.from_numpy(G[f"{run}_face_idx"]))
    for k in ref_keys - {"face_idx"}:
        assert err(res[k], torch.from_numpy(G[f"{run}_{k}"])) <= 1e-5, (k, err(res[k], torch.from_numpy(G[f"{run}_{k}"])))


def test_default_light():
    mats, _ = materials(False)
    m = mesh(mats)
    res = easy_render.render_mesh(camera(m.vertices), m, backend="cuda")
    check_passes(res, "default")
    cov = res["face_idx"] >= 0
    assigned = m.material_assignments[res["face_idx"][cov]]
    assert set(assigned.unique().tolist()) == {0, 1}                # both materials are on screen


def test_lights_and_texture_gradients():
    mats, tex = materials(True)
    m = mesh(mats)
    lp = [T(k).requires_grad_(True) for k in ("light_amp", "light_dir", "light_sharp")]
    lights = types.SimpleNamespace(amplitude=lp[0], direction=lp[1], sharpness=lp[2])
    res = easy_render.render_mesh(camera(m.vertices), m, lighting=lights)
    check_passes(res, "lit")
    (res["render"] * T("w")).sum().backward()
    for k, t in zip(("amp", "dir", "sharp"), lp):
        assert err(t.grad, torch.from_numpy(G[f"lit_g_light_{k}"])) <= 1e-5, k
    for k in ("diffuse_texture", "roughness_texture"):
        assert err(tex[k].grad, torch.from_numpy(G[f"lit_g_m0_{k}"])) <= 1e-5, k


def test_texture_sample_materials_matches_the_rendered_passes():
    mats, _ = materials(False)
    m = mesh(mats)
    cam = camera(m.vertices)
    res = easy_render.render_mesh(cam, m)
    face_idx, base, tangents, uvs, _ = easy_render.mesh_rasterize_interpolate_cuda(m, cam)
    sign = torch.cross(*(T("vertices_ndc")[m.faces][:, k] - T("vertices_ndc")[m.faces][:, 0] for k in (1, 2)),
                       dim=-1)[..., 2]
    s = torch.sign(sign[face_idx]) * (face_idx >= 0)
    albedo, spec_albedo, normals, roughness = easy_render.texture_sample_materials(
        "cuda", face_idx, base * s.unsqueeze(-1), mats, uv_map=uvs, material_assignments=m.material_assignments,
        im_tangents=tangents)
    assert torch.equal(albedo, res["albedo"]) and torch.equal(normals, res["normals"])
    cov = face_idx >= 0
    assert (roughness[cov] >= 1e-3).all() and (roughness[~cov] == 0.5).all()
    assert (spec_albedo[~cov] == 0).all() and (spec_albedo[cov] > 0).any()
