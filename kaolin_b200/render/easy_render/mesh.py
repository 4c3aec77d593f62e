"""Kaolin's one-call renderer (kaolin/render/easy_render/mesh.py) on this library's kernels.

* ``mesh_rasterize_interpolate_cuda`` (mesh.py:141-209): rasterize + interpolate on the H100
  rasterizer (wide feature interpolation: normals 3 + uvs 2 + tangents 3 + features k).
* ``texture_sample_materials`` (mesh.py:278-424): the reference's per-material sampling in torch, with
  this library's ``texture_mapping``.
* ``sg_shade`` (mesh.py:427-464): deferred spherical-Gaussian shading, one fused sm_90a kernel each way
  (kaolin_b200/csrc/lighting.cu, kind SHADE) instead of boolean gathers, a ray grid, two lighting
  passes and six scatters.
* ``render_mesh`` (mesh.py:53-138): the four chained, with the CUDA backend only.

Everything is duck-typed exactly on what the reference functions touch, so a
``kaolin.rep.SurfaceMesh`` / ``kaolin.render.camera.Camera`` / ``PBRMaterial`` /
``SgLightingParameters`` works unchanged, and so does any object exposing the same attributes:

  mesh:     vertices (V,3), faces (F,3) long, face_normals (1,F,3,3) or (F,3,3),
            optional face_uvs (..,F,3,2), face_tangents (..,F,3,3), face_features (..,F,3,k),
            has_attribute(name), has_or_can_compute_attribute(name), as_transformed(),
            materials, material_assignments, len(), [0]
  camera:   extrinsics.transform(points), extrinsics.R, intrinsics.transform(points), transform(points),
            height, width, x0, y0, focal_x, focal_y, dtype, device, len()
  material: chw(), normals/diffuse/specular/metallic/roughness_texture, diffuse_color, specular_color,
            metallic_value, roughness_value, is_specular_workflow
  lighting: amplitude (L,3), direction (L,3), sharpness (L,)
"""
import logging
import math
import warnings

from enum import Enum

import torch
from torch.autograd import Function

from ... import _lib
from ..mesh import _host, rasterize, texture_mapping

__all__ = ["render_mesh", "mesh_rasterize_interpolate_cuda", "texture_sample_materials", "sg_shade", "RenderPass"]

logger = logging.getLogger(__name__)


class RenderPass(str, Enum):
    face_idx = "face_idx"
    uvs = "uvs"
    albedo = "albedo"
    normals = "normals"
    roughness = "roughness"
    diffuse = "diffuse"
    specular = "specular"
    features = "features"
    render = "render"
    alpha = "alpha"


def _index_vertices_by_faces(vertices_features, faces):
    """ops/mesh/mesh.py:54-76 (a gather): (B,V,k), (F,3) -> (B,F,3,k)."""
    return vertices_features[:, faces]


def _face_attr(x):
    return x if x.dim() == 4 else x.unsqueeze(0)


def mesh_rasterize_interpolate_cuda(mesh, camera, normals_required=True, uvs_required=True,
                                    tangents_required=True, features_required=True):
    """Rasterization and interpolation of an unbatched mesh seen by a single camera
    (kaolin/render/easy_render/mesh.py:141-209).  Returns
    ``(face_idx, im_normals, im_tangents, im_uvs, im_features)`` — image-space values at the camera
    resolution for the attributes that are required and available, ``None`` for the others."""
    if mesh.has_attribute('transform'):
        mesh = mesh.as_transformed()
        warnings.warn("Mesh has a transform attribute, transforming to world space. "
                      "If you are rasterizing the mesh multiple times, "
                      "consider transforming it once before rasterizing it.", stacklevel=2)

    vertices_camera = camera.extrinsics.transform(mesh.vertices)
    vertices_image = camera.intrinsics.transform(vertices_camera)
    if vertices_camera.dim() == 2:
        vertices_camera, vertices_image = vertices_camera.unsqueeze(0), vertices_image.unsqueeze(0)

    face_vertices_camera = _index_vertices_by_faces(vertices_camera, mesh.faces)
    face_vertices_image = _index_vertices_by_faces(vertices_image, mesh.faces)[..., :2]

    in_face_features = []
    idx_normals = idx_uvs = idx_tangents = idx_features = -1
    current_idx = 0
    if normals_required:
        in_face_features.append(_face_attr(mesh.face_normals))
        idx_normals = current_idx
        current_idx += in_face_features[-1].shape[-1]
    if uvs_required and mesh.has_or_can_compute_attribute('face_uvs'):
        in_face_features.append(_face_attr(mesh.face_uvs))
        idx_uvs = current_idx
        current_idx += in_face_features[-1].shape[-1]
    if tangents_required and mesh.has_or_can_compute_attribute('face_tangents'):
        in_face_features.append(_face_attr(mesh.face_tangents))
        idx_tangents = current_idx
        current_idx += in_face_features[-1].shape[-1]
    if features_required and mesh.has_or_can_compute_attribute('face_features'):
        in_face_features.append(_face_attr(mesh.face_features))
        idx_features = current_idx
        current_idx += in_face_features[-1].shape[-1]

    if len(in_face_features) == 0:
        in_face_features = [torch.zeros((1,) + tuple(mesh.faces.shape) + (1,), dtype=camera.dtype,
                                        device=camera.device)]

    in_face_features = torch.cat(in_face_features, dim=-1).float()
    face_features, face_idx = rasterize(
        camera.height, camera.width,
        face_features=in_face_features,
        face_vertices_z=face_vertices_camera[..., -1].float().contiguous(),
        face_vertices_image=face_vertices_image.float().contiguous())

    im_normals = im_uvs = im_tangents = im_features = None
    if idx_normals >= 0:
        im_normals = face_features[..., idx_normals:idx_normals + 3]
    if idx_uvs >= 0:
        im_uvs = face_features[..., idx_uvs:idx_uvs + 2] % 1.
    if idx_tangents >= 0:
        im_tangents = face_features[..., idx_tangents:idx_tangents + 3]
    if idx_features >= 0:
        im_features = face_features[..., idx_features:]

    return face_idx, im_normals, im_tangents, im_uvs, im_features


class _Lighting:
    """The default light of easy_render/common.py: one SG of amplitude 3, sharpness 5, from azimuth 2.3
    and elevation pi / 3 (sg_direction_from_azimuth_elevation, y up)."""

    def __init__(self, device):
        azimuth = torch.full((1,), 2.3, dtype=torch.float)
        elevation = torch.full((1,), math.pi / 3., dtype=torch.float)
        temp = torch.cos(elevation)
        direction = torch.stack([torch.sin(azimuth) * temp, torch.sin(elevation), torch.cos(azimuth) * temp], dim=-1)
        self.amplitude = torch.full((1, 3), 3., device=device)
        self.direction = torch.nn.functional.normalize(direction.reshape(-1, 3), dim=1).to(device)
        self.sharpness = torch.full((1,), 5., device=device)


class _Material:
    """The default material of easy_render/common.py: green diffuse, specular colour (0.7, 0.5, 0.7),
    specular workflow, no textures."""
    normals_texture = diffuse_texture = specular_texture = metallic_texture = roughness_texture = None
    metallic_value = roughness_value = None
    is_specular_workflow = True

    def __init__(self, device):
        self.diffuse_color = torch.tensor((118.0 / 255.0, 185.0 / 255.0, 0.), device=device)
        self.specular_color = torch.tensor((0.7, 0.5, 0.7), device=device)

    def chw(self):
        return self


def _texture_sample_material_cuda(material, texcoords):
    """The material's texture maps at ``texcoords`` (1,1,N,2), one texture_mapping call for all the maps
    of the first map's size (easy_render/mesh.py:_texture_sample_material_cuda)."""
    def _texture_map(_texcoords, _image):
        return texture_mapping(_texcoords, _image.unsqueeze(0).contiguous(), mode='bilinear').squeeze(0).squeeze(0)

    texture_images = []
    current_idx = 0
    name_idx_nchannels = {}
    for name, image in zip(['normals', 'diffuse', 'specular', 'metalic', 'roughness'],
                           [material.normals_texture, material.diffuse_texture, material.specular_texture,
                            material.metallic_texture, material.roughness_texture]):
        if image is not None:
            if len(texture_images) == 0 or texture_images[0].shape[-2:] == image.shape[-2:]:
                texture_images.append(image)
                name_idx_nchannels[name] = (current_idx, image.shape[-3])
                current_idx += image.shape[-3]
            else:
                name_idx_nchannels[name] = _texture_map(texcoords, image.float())
        else:
            name_idx_nchannels[name] = (-1, 0)

    rendered_images = None
    if len(texture_images) > 0:
        rendered_images = _texture_map(texcoords, torch.cat(texture_images, dim=-3).float())

    def _proc_attr(name):
        preproc = name_idx_nchannels[name]
        if torch.is_tensor(preproc):
            return preproc
        idx, nchannels = preproc
        return rendered_images[..., idx:idx + nchannels] if idx >= 0 else None

    return tuple(_proc_attr(n) for n in ('normals', 'diffuse', 'specular', 'metalic', 'roughness'))


def texture_sample_materials(backend, face_idx, im_base_normals, materials=None, uv_map=None,
                             material_assignments=None, im_tangents=None):
    """Image-space material channels of a rasterized mesh (easy_render/mesh.py:278-424):
    ``(albedo, spec_albedo, im_world_normals, im_roughness)``, (B,H,W,3) x 3 and (B,H,W,1).  Per
    material: its texture maps (or constant values) where ``material_assignments[face_idx]`` selects it,
    the tangent-space normal map applied to ``im_base_normals``, the metallic-roughness workflow turned
    into diffuse and specular albedo (glTF 2.0), roughness clamped at 1e-3.  Background pixels keep 0
    (roughness 0.5).  Only the ``'cuda'`` backend is provided.  Each material costs one host
    synchronisation (whether it is visible), as in the reference."""
    if backend == 'nvdiffrast':
        raise ValueError('kaolin_b200: the "nvdiffrast" backend is not provided; use backend="cuda"')
    if backend != 'cuda':
        raise ValueError(f'Unsupported backend {backend}, "nvdiffrast" and "cuda" are supported.')
    batch, height, width = face_idx.shape[0], face_idx.shape[-2], face_idx.shape[-1]
    device = face_idx.device

    albedo = torch.zeros((batch, height, width, 3), device=device)
    spec_albedo = torch.zeros((batch, height, width, 3), device=device)
    im_world_normals = torch.zeros((batch, height, width, 3), device=device)
    im_roughness = torch.zeros((batch, height, width, 1), device=device) + 0.5

    if materials is None:
        materials = [_Material(device)]

    if material_assignments is not None:
        im_material_idx = material_assignments[face_idx]
    else:
        im_material_idx = torch.zeros((batch, height, width), dtype=torch.int16, device=device)
    im_material_idx[face_idx == -1] = -1

    im_bitangents = None
    if im_tangents is not None and im_base_normals is not None:
        im_bitangents = torch.nn.functional.normalize(torch.cross(im_tangents, im_base_normals, dim=-1), dim=-1)

    for i, material in enumerate(materials):
        mask = im_material_idx == i
        if mask.count_nonzero().item() == 0:
            continue

        perturbation_normal = mapped_albedo = mapped_spec = mapped_metalic = mapped_roughness = None
        if uv_map is None:
            logger.warning('Missing uvmap; cannot texturemap materials')
        else:
            texcoords = uv_map[mask].reshape(1, 1, -1, 2).contiguous()
            texcoords[..., 1] = 1 - texcoords[..., 1]
            perturbation_normal, mapped_albedo, mapped_spec, mapped_metalic, mapped_roughness = \
                _texture_sample_material_cuda(material.chw(), texcoords)

        if perturbation_normal is not None and im_tangents is not None and im_bitangents is not None:
            perturbation_normal = perturbation_normal.unsqueeze(0).unsqueeze(0)
            im_world_normals[mask] = torch.nn.functional.normalize(
                im_tangents[mask] * perturbation_normal[..., :1]
                - im_bitangents[mask] * perturbation_normal[..., 1:2]
                + im_base_normals[mask] * perturbation_normal[..., 2:3], dim=-1)
        else:
            im_world_normals[mask] = im_base_normals[mask]

        if mapped_albedo is not None:
            albedo[mask] = mapped_albedo[..., :3]
        elif material.diffuse_color is not None:
            albedo[mask] = material.diffuse_color.unsqueeze(0)

        if material.is_specular_workflow:
            if mapped_spec is not None:
                spec_albedo[mask] = mapped_spec
            elif material.specular_color is not None:
                spec_albedo[mask] = material.specular_color.unsqueeze(0)
        else:
            metalic_val = mapped_metalic if mapped_metalic is not None else material.metallic_value
            if metalic_val is not None:
                spec_albedo[mask] = (1. - metalic_val) * 0.04 + albedo[mask] * metalic_val
                albedo[mask] = albedo[mask] * (1. - metalic_val)

        if mapped_roughness is not None:
            im_roughness[mask] = mapped_roughness.clamp(min=1e-3)
        elif material.roughness_value is not None:
            im_roughness[mask] = material.roughness_value.unsqueeze(0).clamp(min=1e-3)

    return albedo, spec_albedo, im_world_normals, im_roughness


def _camera_block(camera):
    """(C, 16) float32 on the camera's device, built with torch ops (no host round trip): R row-major,
    tan_x, tan_y, x0, y0, camera width, camera height, 0.  tan_* as Camera.tan_half_fov computes them."""
    R = camera.extrinsics.R
    fx, fy, x0, y0 = camera.focal_x, camera.focal_y, camera.x0, camera.y0
    C = R.shape[0]
    tan_x = torch.full_like(fx, camera.width / 2.0) / fx
    tan_y = torch.full_like(fy, camera.height / 2.0) / fy
    size = torch.zeros((C, 3), dtype=torch.float32, device=R.device)     # fills only: no host copy
    size[:, 0] = float(camera.width)
    size[:, 1] = float(camera.height)
    cols = [R.reshape(C, 9), tan_x.reshape(C, 1), tan_y.reshape(C, 1), x0.reshape(C, 1), y0.reshape(C, 1), size]
    return torch.cat([c.to(torch.float32) for c in cols], dim=1).contiguous()


class SgShadeB200(Function):
    """sg_shade of a (B,H,W) G-buffer: one SHADE kernel each way."""

    @staticmethod
    def forward(ctx, cam, face_idx, albedo, spec_albedo, roughness, normals, amplitude, direction, sharpness):
        ins = [t.contiguous() for t in (face_idx, albedo, spec_albedo, roughness, normals,
                                        amplitude, direction, sharpness)]
        B, H, W = face_idx.shape
        diffuse, specular, img = (torch.empty((B, H, W, 3), dtype=torch.float32, device=albedo.device)
                                  for _ in range(3))
        _lib.call("dibr_b200_sg_shade_forward", albedo.device,
                  B, H, W, amplitude.shape[0], cam, *ins, diffuse, specular, img)
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(cam, *ins)
        return diffuse, specular, img

    @staticmethod
    def backward(ctx, g_diffuse, g_specular, g_img):
        cam, face_idx, albedo, spec_albedo, roughness, normals, amplitude, direction, sharpness = ctx.saved_tensors
        wants = ctx.needs_input_grad[2:]
        grads = [torch.empty_like(t) if w else None
                 for t, w in zip((albedo, spec_albedo, roughness, normals, amplitude, direction, sharpness), wants)]
        if all(g is None for g in (g_diffuse, g_specular, g_img)) or not any(wants):
            return (None, None) + tuple(None if g is None else g.zero_() for g in grads)
        B, H, W = face_idx.shape
        L = amplitude.shape[0]
        dev = albedo.device
        ws = _lib.scratch(_lib.lib().dibr_b200_sg_shade_workspace_bytes(L) if any(wants[4:]) else 0, dev)
        gouts = [None if g is None else g.contiguous() for g in (g_diffuse, g_specular, g_img)]
        _lib.call("dibr_b200_sg_shade_backward", dev,
                  B, H, W, L, cam, face_idx, albedo, spec_albedo, roughness, normals, amplitude, direction, sharpness,
                  *gouts, *grads, ws, ws.numel())
        return (None, None) + tuple(grads)


def sg_shade(camera, face_idx, albedo, spec_albedo, im_roughness, im_world_normals, amplitude, direction, sharpness):
    """Partial PBR shading of image-space material maps under spherical-Gaussian lights
    (easy_render/mesh.py:427-464): ``(diffuse_img, specular_img, img)``, each (B,H,W,3) float32.

    ``face_idx`` (B,H,W) int64 marks the covered pixels (>= 0); ``albedo``, ``spec_albedo`` and
    ``im_world_normals`` are (B,H,W,3) and ``im_roughness`` (B,H,W,1); lights are ``amplitude`` (L,3),
    ``direction`` (L,3) and ``sharpness`` (L,).  The diffuse term is ``sg_diffuse_inner_product`` and the
    specular term ``sg_warp_specular_term`` of the normalised normal, with the view towards the camera
    through each pixel of the custom-resolution grid of ``camera`` (``len(camera) == B``; the reference
    takes B = 1).  Background pixels are 0.  One kernel each way, no host synchronisation; gradients flow
    to the maps and the lights (bit-reproducible), not to the camera."""
    cam_tensors = (camera.extrinsics.R, camera.x0, camera.y0, camera.focal_x, camera.focal_y)
    if torch.is_grad_enabled() and any(t.requires_grad for t in cam_tensors):
        raise NotImplementedError("sg_shade: gradients to the camera are not implemented; "
                                  "detach the camera parameters")
    tensors = [("face_idx", face_idx), ("albedo", albedo), ("spec_albedo", spec_albedo),
               ("im_roughness", im_roughness), ("im_world_normals", im_world_normals), ("amplitude", amplitude),
               ("direction", direction), ("sharpness", sharpness)]
    _host.check_tensors("sg_shade", tensors)
    if face_idx.dtype != torch.int64:
        raise RuntimeError(f"sg_shade: expected face_idx to be int64, got {face_idx.dtype}")
    assert face_idx.dim() == 3, face_idx.shape
    B, H, W = face_idx.shape
    assert albedo.shape == (B, H, W, 3) and spec_albedo.shape == (B, H, W, 3), (albedo.shape, spec_albedo.shape)
    assert im_world_normals.shape == (B, H, W, 3), im_world_normals.shape
    assert im_roughness.shape in ((B, H, W, 1), (B, H, W)), im_roughness.shape
    assert amplitude.ndim == 2 and amplitude.shape[1] == 3
    assert direction.shape == amplitude.shape and sharpness.shape == amplitude.shape[:1]
    if len(camera) != B:
        raise ValueError(f"sg_shade: the camera has {len(camera)} views, face_idx has {B}")
    cam = _camera_block(camera)
    _host.check_tensors("sg_shade", [("albedo", albedo), ("camera", cam)])     # the camera's device
    return SgShadeB200.apply(cam, face_idx, albedo, spec_albedo, im_roughness, im_world_normals,
                             amplitude, direction, sharpness)


def render_mesh(camera, mesh, lighting=None, custom_materials=None, custom_material_assignments=None,
                backend=None, nvdiffrast_context=None):
    """Kaolin's default differentiable renderer (easy_render/mesh.py:53-138) for one camera and one
    mesh: rasterize + interpolate, the reference's face-normal sign flip, material sampling and the
    fused ``sg_shade``.  Returns a dict from ``RenderPass`` names to (1,H,W,C) images; it always holds
    ``'render'``.  Only the ``'cuda'`` backend is provided (``None`` selects it)."""
    if len(camera) != 1:
        raise NotImplementedError('Render is only implemented for single unbatched camera.')
    if len(mesh) > 1:
        raise NotImplementedError(f'Render is only implemented for mesh of length 1, not {len(mesh)}.')
    mesh = mesh[0]
    if mesh.has_attribute('transform'):
        mesh = mesh.as_transformed()
        warnings.warn("Mesh has a transform attribute, transforming to world space. "
                      "If you are rasterizing the mesh multiple times, "
                      "consider transforming it once before rasterizing it.", stacklevel=2)
    if backend is None:
        backend = "cuda"
    if backend == "nvdiffrast":
        raise ValueError('kaolin_b200: the "nvdiffrast" backend is not provided; use backend="cuda"')
    if backend != "cuda":
        raise ValueError(f'Unsupported backend {backend}, "nvdiffrast" and "cuda" are supported.')

    materials = custom_materials or mesh.materials
    material_assignments = custom_material_assignments if custom_material_assignments is not None \
        else mesh.material_assignments
    if lighting is None:
        lighting = _Lighting(camera.device)

    face_idx, im_base_normals, im_tangents, uv_map, im_features = mesh_rasterize_interpolate_cuda(mesh, camera)

    if im_base_normals is not None:
        face_vertices_ndc = _index_vertices_by_faces(camera.transform(mesh.vertices).unsqueeze(0), mesh.faces)
        e0 = face_vertices_ndc[:, :, 1] - face_vertices_ndc[:, :, 0]
        e1 = face_vertices_ndc[:, :, 2] - face_vertices_ndc[:, :, 0]
        face_normal_sign = torch.cross(e0, e1, dim=2)[..., 2]
        im_normal_sign = torch.sign(face_normal_sign[0, face_idx])
        im_normal_sign[face_idx == -1] = 0.
        im_base_normals = im_base_normals * im_normal_sign.unsqueeze(-1)

    albedo, spec_albedo, im_world_normals, im_roughness = texture_sample_materials(
        backend, face_idx, im_base_normals, materials,
        uv_map=uv_map, material_assignments=material_assignments, im_tangents=im_tangents)

    diffuse_img, specular_img, img = sg_shade(
        camera, face_idx, albedo, spec_albedo, im_roughness, im_world_normals,
        lighting.amplitude, lighting.direction, lighting.sharpness)

    res = {
        RenderPass.face_idx.name: face_idx,
        RenderPass.render.name: img,
        RenderPass.albedo.name: albedo,
        RenderPass.normals.name: im_world_normals,
        RenderPass.diffuse.name: diffuse_img,
        RenderPass.specular.name: specular_img,
        RenderPass.uvs.name: uv_map,
        RenderPass.features.name: im_features,
    }
    return {k: v for k, v in res.items() if v is not None}
