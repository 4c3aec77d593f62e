"""``prepare_vertices`` and ``texture_mapping`` — drop-ins for kaolin/render/mesh/utils.py:22-79
and :129-175, the steps immediately before and after the rasterizer in every DIB-R caller
(SURVEY.md §8f rank 1 and 2).  One sm_90a kernel each way (kaolin_b200/csrc/mesh_pipeline.cu)
instead of the reference's chain of PyTorch kernels and its (B,V,3)/(B,V,2) intermediates.
Same signatures, argument meaning and return structure; CUDA tensors only (no CPU path).
"""
import ctypes

import torch
from torch.autograd import Function

from ... import _lib
from . import _host

__all__ = ["prepare_vertices", "texture_mapping"]


def _proj3(camera_proj):
    """camera_proj (3,1) -> host array of 3 floats (one tiny D2H if it lives on the GPU, as the
    reference's broadcast would read it on the device)."""
    vals = [float(x) for x in camera_proj.detach().reshape(-1).tolist()]
    if len(vals) != 3:
        raise RuntimeError("prepare_vertices: camera_proj must be of shape (3, 1)")
    return (ctypes.c_float * 3)(*vals)


class PrepareVerticesB200(Function):
    @staticmethod
    def forward(ctx, vertices, faces, camera_proj, camera_rot, camera_trans, camera_transform):
        # an output the loss does not use arrives in backward as None (a NULL pointer: the kernel
        # skips that branch) instead of a tensor of zeros it would read and multiply through
        ctx.set_materialize_grads(False)
        v = vertices.contiguous()
        f = faces.contiguous()
        B, V = v.shape[0], v.shape[1]
        F = f.shape[0]
        T = None if camera_transform is None else camera_transform.contiguous()
        R = None if camera_rot is None else camera_rot.contiguous()
        t = None if camera_trans is None else camera_trans.reshape(B, 3).contiguous()
        proj = _proj3(camera_proj)
        fvc = torch.empty((B, F, 3, 3), dtype=torch.float32, device=v.device)
        fvi = torch.empty((B, F, 3, 2), dtype=torch.float32, device=v.device)
        fn = torch.empty((B, F, 3), dtype=torch.float32, device=v.device)
        if F:       # an empty mesh has empty outputs (and no storage to point the kernel at)
            _lib.call("dibr_b200_prepare_vertices_forward", v.device, B, V, F, v, f, T, R, t, proj, fvc, fvi, fn)
        ctx.save_for_backward(v, f, T, R, t)
        ctx.proj = proj
        ctx.trans_shape = None if camera_trans is None else camera_trans.shape     # (B, 3) or (B, 1, 3)
        return fvc, fvi, fn

    @staticmethod
    def backward(ctx, g_fvc, g_fvi, g_fn):
        v, f, T, R, t = ctx.saved_tensors
        B, V = v.shape[0], v.shape[1]
        F = f.shape[0]
        c = lambda g: None if g is None else g.contiguous()
        g_fvc, g_fvi, g_fn = c(g_fvc), c(g_fvi), c(g_fn)
        g_vc = (torch.empty if F else torch.zeros)((B, V, 3), dtype=torch.float32, device=v.device)
        if F:
            _lib.call("dibr_b200_prepare_vertices_backward", v.device,
                      B, V, F, v, f, T, R, t, ctx.proj, g_fvc, g_fvi, g_fn, g_vc)
        # the camera map is linear: back through it with library GEMMs ((B,V,3) x (3,3))
        g_v = g_T = g_R = g_t = None
        if T is not None:
            if ctx.needs_input_grad[0]:
                g_v = g_vc @ T[:, :3, :].transpose(1, 2)
            if ctx.needs_input_grad[5]:
                g_T = torch.cat([v.transpose(1, 2) @ g_vc, g_vc.sum(dim=1, keepdim=True)], dim=1)
        else:
            g_d = g_vc @ R                        # vc = (p - t) @ R^T
            if ctx.needs_input_grad[0]:
                g_v = g_d
            if ctx.needs_input_grad[3]:
                g_R = g_vc.transpose(1, 2) @ (v - t.view(B, 1, 3))
            if ctx.needs_input_grad[4]:
                g_t = -g_d.sum(dim=1).view(ctx.trans_shape)
        return g_v, None, None, g_R, g_t, g_T


def prepare_vertices(vertices, faces, camera_proj, camera_rot=None, camera_trans=None,
                     camera_transform=None):
    r"""Move and project vertices to the cameras, then index them with faces
    (kaolin.render.mesh.utils.prepare_vertices, utils.py:129-175).

    Returns ``(face_vertices_camera (B,F,3,3), face_vertices_image (B,F,3,2), face_normals (B,F,3))``.
    Gradients flow to ``vertices`` and to the camera transform / rotation / translation;
    ``camera_proj`` is treated as a constant.

    ``vertices`` and the camera tensors must be float32 and ``faces`` int64; any other element
    type, integer and bool included, raises.  ``camera_trans`` may be (B, 3) or (B, 1, 3).
    A face of zero area ((a, a, b), three collinear vertices) gets the normal 0 and, as the
    reference's ``norm`` subgradient does, passes no normal gradient to its vertices.  A vertex
    on the camera plane (z = 0) gives inf / NaN image coordinates on the faces that use it, as in
    the reference, and on no other face.  The entries of ``faces`` are not range-checked: an index
    outside [0, num_vertices) is read as it is (``kaolin_b200.ops.mesh`` raises IndexError for the
    same mistake, at the cost of a host synchronisation this call does not make).
    """
    if camera_transform is None:
        assert camera_trans is not None and camera_rot is not None, \
            "camera_transform or camera_trans and camera_rot must be defined"
    else:
        assert camera_trans is None and camera_rot is None, \
            "camera_trans and camera_rot must be None when camera_transform is defined"
    _host.check_tensors("prepare_vertices", [("vertices", vertices), ("faces", faces),
                                             ("camera_rot", camera_rot), ("camera_trans", camera_trans),
                                             ("camera_transform", camera_transform)])
    _host.check_float32("prepare_vertices", [("vertices", vertices), ("camera_rot", camera_rot),
                                             ("camera_trans", camera_trans),
                                             ("camera_transform", camera_transform)])
    if vertices.dim() != 3 or vertices.shape[-1] != 3:
        raise RuntimeError("prepare_vertices: vertices must be of shape (batch_size, num_vertices, 3)")
    if faces.dim() != 2 or faces.shape[-1] != 3 or faces.dtype != torch.int64:
        raise NotImplementedError("prepare_vertices: faces must be a LongTensor of shape (num_faces, 3) "
                                  "(triangle meshes)")
    B = vertices.shape[0]
    if camera_transform is not None:
        _host.check_size("prepare_vertices", "camera_transform", camera_transform, (B, 4, 3))
    else:
        _host.check_size("prepare_vertices", "camera_rot", camera_rot, (B, 3, 3))
        if camera_trans.numel() != B * 3:
            raise RuntimeError("prepare_vertices: camera_trans must hold (batch_size, 3) values")
    return PrepareVerticesB200.apply(vertices, faces, camera_proj, camera_rot, camera_trans, camera_transform)


class TextureMappingB200(Function):
    @staticmethod
    def forward(ctx, texture_coordinates, texture_maps, nearest):
        uv = texture_coordinates.contiguous()
        if uv.data_ptr() % 8:       # the kernels load (u, v) as one float2; a contiguous view at an odd
            uv = uv.clone()         # element offset is legal input and is not copied by contiguous()
        tex = texture_maps.contiguous()
        B, C, Ht, Wt = tex.shape
        N = uv.numel() // (2 * B)
        out = torch.empty((B, N, C), dtype=torch.float32, device=uv.device)
        if N:       # no points: an empty output (and no storage to point the kernel at)
            _lib.call("dibr_b200_texture_mapping_forward", uv.device, B, N, C, Ht, Wt, uv, tex, int(nearest), out)
        ctx.save_for_backward(uv, tex)
        ctx.nearest = int(nearest)
        return out

    @staticmethod
    def backward(ctx, g_out):
        uv, tex = ctx.saved_tensors
        B, C, Ht, Wt = tex.shape
        N = uv.numel() // (2 * B)
        g_tex = torch.empty_like(tex) if ctx.needs_input_grad[1] else None
        g_uv = torch.empty_like(uv) if ctx.needs_input_grad[0] else None
        if N:
            _lib.call("dibr_b200_texture_mapping_backward", uv.device,
                      B, N, C, Ht, Wt, uv, tex, ctx.nearest, g_out.contiguous(), g_tex, g_uv)
        elif g_tex is not None:
            g_tex.zero_()
        return g_uv, g_tex, None


def texture_mapping(texture_coordinates, texture_maps, mode='nearest'):
    r"""Interpolates ``texture_maps`` (B,C,h',w') at dense (B,h,w,2) or sparse (B,N,2) OpenGL texture
    coordinates in [0,1] (kaolin.render.mesh.utils.texture_mapping, utils.py:22-79): clamp,
    y flip, ``grid_sample(align_corners=False, padding_mode='border')``.  ``mode``: 'nearest'
    or 'bilinear'.  Returns (B,h,w,C) or (B,N,C).

    Both arguments must be float32; any other element type, integer and bool included, raises.
    'nearest' rounds half to even, as ``grid_sample`` does, and gives the coordinates a zero
    gradient.  In 'bilinear' the coordinate gradient is zero where the clamp to [0, 1] or the
    border clip acts: outside the open interval (0, 1) and within half a texel of either edge.
    +-inf clamp like any other value.  One deliberate difference from the reference: a NaN
    coordinate is read as 0 (u: the leftmost column, v: the bottom row) and gets a zero gradient,
    where ``grid_sample`` propagates the NaN and what it then samples differs between its CPU and
    CUDA kernels and between forward and backward."""
    if mode not in ('nearest', 'bilinear'):
        raise ValueError(f"texture_mapping: mode must be 'nearest' or 'bilinear', got '{mode}'")
    _host.check_tensors("texture_mapping", [("texture_coordinates", texture_coordinates),
                                            ("texture_maps", texture_maps)])
    _host.check_float32("texture_mapping", [("texture_coordinates", texture_coordinates),
                                            ("texture_maps", texture_maps)])
    if texture_maps.dim() != 4 or texture_coordinates.shape[-1] != 2 \
            or texture_coordinates.shape[0] != texture_maps.shape[0]:
        raise RuntimeError("texture_mapping: expected texture_coordinates (B,...,2) and texture_maps (B,C,h',w')")
    out = TextureMappingB200.apply(texture_coordinates, texture_maps, mode == 'nearest')
    return out.reshape(texture_coordinates.shape[0], *texture_coordinates.shape[1:-1], texture_maps.shape[1])
