"""``kaolin_b200._C.render.mesh`` — the four operators the reference registers in
kaolin/csrc/bindings.cpp:111-115, with identical names, argument order/meaning,
return structure and error behaviour, implemented by libdibr_b200.so; likewise
``_C.render.sg``, the DefTet pair, ``_C.ops.mesh.unbatched_mesh_intersection_cuda``
(bindings.cpp:49), which the reference's ``check_sign.py`` calls, and
``_C.ops.conversions.unbatched_mcube_forward_cuda``, which its ``voxelgrids_to_trianglemeshes`` calls, and
``_C.metrics.unbatched_triangle_distance_{forward,backward}_cuda``, which its ``point_to_mesh_distance`` calls.

This is what makes the library a drop-in *below* the reference's own Python
wrappers: ``kaolin.render.mesh.rasterization`` / ``.dibr`` run unmodified with
``kaolin._C`` replaced by this module (tests/test_reference_wrappers.py: arity / dispatch on CPU,
results on the GPU).
"""
import types

import torch

from . import _lib
from .render.mesh import _host


def _check_all(func, named, float_dtype=torch.float32):
    """at::checkAllSameGPU + at::checkAllContiguous (rasterization.cpp:70-75)."""
    dev = None
    for name, t in named:
        if not t.is_cuda:
            raise RuntimeError(f"{func}: expected tensor for argument {name} to be on GPU "
                               "(kaolin_b200 has no CPU path)")
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise RuntimeError(f"{func}: expected all tensors on the same GPU; {name} is on {t.device}")
        if not t.is_contiguous():
            raise RuntimeError(f"{func}: expected contiguous tensor for argument {name}")
        if t.is_floating_point() and t.dtype != float_dtype:
            raise RuntimeError(f"\"{func}\" not implemented for '{str(t.dtype).replace('torch.', '')}' "
                               "(kaolin_b200 supports float32)")
    return dev


def _fp64_via_fp32(op):
    """The reference's operators dispatch float and double (AT_DISPATCH_FLOATING_TYPES,
    rasterization_cuda.cu:218/427, dibr_soft_mask_cuda.cu:205/376).  The public API has a real
    <double> instantiation (render/mesh/dibr.py:DibrRasterizationB200 -> dibr_b200_forward_f64); these
    packed operator shims serve double callers by casting: float64 inputs -> float32, the op,
    floating-point outputs -> float64 (fp32 rounding applies)."""
    import functools

    @functools.wraps(op)
    def wrapped(*args):
        if not any(isinstance(a, torch.Tensor) and a.dtype == torch.float64 for a in args):
            return op(*args)
        out = op(*[a.to(torch.float32) if isinstance(a, torch.Tensor) and a.dtype == torch.float64 else a
                   for a in args])
        cast = lambda t: t.to(torch.float64) if isinstance(t, torch.Tensor) and t.dtype == torch.float32 else t
        return [cast(t) for t in out] if isinstance(out, (list, tuple)) else cast(out)
    return wrapped


def _check_size(func, name, t, shape):
    if tuple(t.shape) != tuple(shape):
        raise RuntimeError(f"{func}: expected tensor of size {list(shape)} for argument {name}, "
                           f"got {list(t.shape)}")


@_fp64_via_fp32
def packed_rasterize_forward_cuda(height, width, face_vertices_z, face_vertices_image,
                                  face_bboxes, face_features, first_idx_face_per_mesh,
                                  multiplier, eps):
    """rasterization.cpp:49-104 -> [interpolated_features, selected_face_idx, output_weights]."""
    fn = "packed_rasterize_forward_cuda"
    dev = _check_all(fn, [("face_vertices_z", face_vertices_z),
                          ("face_vertices_image", face_vertices_image),
                          ("face_bboxes", face_bboxes), ("face_features", face_features),
                          ("first_idx_face_per_mesh", first_idx_face_per_mesh)])
    num_faces = face_vertices_z.shape[0]
    batch_size = first_idx_face_per_mesh.shape[0] - 1
    feat_dim = face_features.shape[2]
    _check_size(fn, "face_vertices_z", face_vertices_z, (num_faces, 3))
    _check_size(fn, "face_vertices_image", face_vertices_image, (num_faces, 3, 2))
    _check_size(fn, "face_bboxes", face_bboxes, (num_faces, 4))
    _check_size(fn, "face_features", face_features, (num_faces, 3, feat_dim))
    _check_size(fn, "first_idx_face_per_mesh", first_idx_face_per_mesh, (batch_size + 1,))
    if first_idx_face_per_mesh.dtype != torch.int64:
        raise RuntimeError(f"{fn}: first_idx_face_per_mesh must be a LongTensor")
    idx = torch.empty((batch_size, height, width), dtype=torch.int64, device=dev)
    w = torch.empty((batch_size, height, width, 3), dtype=torch.float32, device=dev)
    out = torch.empty((batch_size, height, width, feat_dim), dtype=torch.float32, device=dev)
    ws = _host.workspace(batch_size, num_faces, height, width, dev)
    _lib.call("dibr_b200_packed_rasterize_forward", dev,
              batch_size, num_faces, height, width, feat_dim, face_vertices_z,
              face_vertices_image, face_bboxes, face_features,
              first_idx_face_per_mesh, float(multiplier), float(eps),
              out, idx, w, ws, ws.numel(), what=fn)
    return [out, idx, w]


@_fp64_via_fp32
def rasterize_backward_cuda(grad_interpolated_features, interpolated_features, selected_face_idx,
                            output_weights, face_vertices_image, face_features, eps):
    """rasterization.cpp:106-168 -> [grad_face_vertices_image, grad_face_features]."""
    fn = "rasterize_backward_cuda"
    dev = _check_all(fn, [("grad_interpolated_features", grad_interpolated_features),
                          ("interpolated_features", interpolated_features),
                          ("selected_face_idx", selected_face_idx),
                          ("output_weights", output_weights),
                          ("face_vertices_image", face_vertices_image),
                          ("face_features", face_features)])
    B, H, W, D = grad_interpolated_features.shape
    F = face_vertices_image.shape[1]
    _check_size(fn, "interpolated_features", interpolated_features, (B, H, W, D))
    _check_size(fn, "selected_face_idx", selected_face_idx, (B, H, W))
    _check_size(fn, "output_weights", output_weights, (B, H, W, 3))
    _check_size(fn, "face_vertices_image", face_vertices_image, (B, F, 3, 2))
    _check_size(fn, "face_features", face_features, (B, F, 3, D))
    g_xy = torch.empty_like(face_vertices_image)
    g_ff = torch.empty_like(face_features)
    # dibr_b200_rasterize_backward shares the fused backward's 16-byte pointer alignment requirement
    (grad_interpolated_features, selected_face_idx, output_weights, face_vertices_image, face_features) = map(
        _host.aligned, (grad_interpolated_features, selected_face_idx, output_weights, face_vertices_image, face_features))
    _lib.call("dibr_b200_rasterize_backward", dev,
              B, F, H, W, D, grad_interpolated_features, selected_face_idx,
              output_weights, face_vertices_image, face_features, float(eps),
              g_xy, g_ff, what=fn)
    return [g_xy, g_ff]


@_fp64_via_fp32
def dibr_soft_mask_forward_cuda(face_vertices_image, face_large_bboxes, selected_face_idx,
                                sigmainv, knum, multiplier):
    """dibr_soft_mask.cpp:48-108 -> [soft_mask, close_face_prob, close_face_idx, close_face_dist_type]."""
    fn = "dibr_soft_mask_forward_cuda"
    dev = _check_all(fn, [("face_vertices_image", face_vertices_image),
                          ("face_bboxes", face_large_bboxes),
                          ("selected_face_idx", selected_face_idx)])
    B, F = face_vertices_image.shape[0], face_vertices_image.shape[1]
    H, W = selected_face_idx.shape[1], selected_face_idx.shape[2]
    _check_size(fn, "face_vertices_image", face_vertices_image, (B, F, 3, 2))
    _check_size(fn, "face_bboxes", face_large_bboxes, (B, F, 4))
    _check_size(fn, "selected_face_idx", selected_face_idx, (B, H, W))
    soft = torch.empty((B, H, W), dtype=torch.float32, device=dev)
    prob = torch.empty((B, H, W, knum), dtype=torch.float32, device=dev)
    cidx = torch.empty((B, H, W, knum), dtype=torch.int64, device=dev)
    ctype = torch.empty((B, H, W, knum), dtype=torch.uint8, device=dev)
    ws = _host.workspace(B, B * F, H, W, dev)
    _lib.call("dibr_b200_soft_mask_forward", dev,
              B, F, H, W, int(knum), face_vertices_image, face_large_bboxes,
              selected_face_idx, float(sigmainv), float(multiplier),
              soft, prob, cidx, ctype, ws, ws.numel(), what=fn)
    return [soft, prob, cidx, ctype]


@_fp64_via_fp32
def dibr_soft_mask_backward_cuda(grad_soft_mask, soft_mask, selected_face_idx, close_face_prob,
                                 close_face_idx, close_face_dist_type, face_vertices_image,
                                 sigmainv, multiplier):
    """dibr_soft_mask.cpp:110-183 -> grad_face_vertices_image."""
    fn = "dibr_soft_mask_backward_cuda"
    dev = _check_all(fn, [("grad_soft_mask", grad_soft_mask), ("soft_mask", soft_mask),
                          ("close_face_idx", close_face_idx),
                          ("close_face_dist_type", close_face_dist_type),
                          ("close_face_prob", close_face_prob),
                          ("face_vertices_image", face_vertices_image)])
    B, F = face_vertices_image.shape[0], face_vertices_image.shape[1]
    H, W = selected_face_idx.shape[1], selected_face_idx.shape[2]
    K = close_face_idx.shape[-1]
    _check_size(fn, "grad_soft_mask", grad_soft_mask, (B, H, W))
    _check_size(fn, "soft_mask", soft_mask, (B, H, W))
    _check_size(fn, "selected_face_idx", selected_face_idx, (B, H, W))
    _check_size(fn, "close_face_prob", close_face_prob, (B, H, W, K))
    _check_size(fn, "close_face_idx", close_face_idx, (B, H, W, K))
    _check_size(fn, "close_face_dist_type", close_face_dist_type, (B, H, W, K))
    _check_size(fn, "face_vertices_image", face_vertices_image, (B, F, 3, 2))
    g = torch.empty_like(face_vertices_image)
    sel = selected_face_idx.contiguous()
    _lib.call("dibr_b200_soft_mask_backward", dev,
              B, F, H, W, K, grad_soft_mask, soft_mask, sel, close_face_prob,
              close_face_idx, close_face_dist_type, face_vertices_image,
              float(sigmainv), float(multiplier), g, what=fn)
    return g


@_fp64_via_fp32
def deftet_sparse_render_forward_cuda(face_vertices_z, face_vertices_image, face_bboxes, pixel_coords,
                                      pixel_depth_ranges, knum, eps):
    """deftet.cpp:48-113 -> [selected_face_idx, pixel_depths, w0_arr, w1_arr], each (B, P, knum)."""
    fn = "deftet_sparse_render_forward_cuda"
    dev = _check_all(fn, [("face_vertices_z", face_vertices_z), ("face_vertices_image", face_vertices_image),
                          ("face_bboxes", face_bboxes), ("pixel_coords", pixel_coords),
                          ("pixel_depth_ranges", pixel_depth_ranges)])
    B, F = face_vertices_z.shape[0], face_vertices_z.shape[1]
    P = pixel_coords.shape[1]
    _check_size(fn, "face_vertices_z", face_vertices_z, (B, F, 3))
    _check_size(fn, "face_vertices_image", face_vertices_image, (B, F, 3, 2))
    _check_size(fn, "face_bboxes", face_bboxes, (B, F, 4))
    _check_size(fn, "pixel_coords", pixel_coords, (B, P, 2))
    _check_size(fn, "pixel_depth_ranges", pixel_depth_ranges, (B, P, 2))
    idx = torch.empty((B, P, knum), dtype=torch.int64, device=dev)
    depth = torch.empty((B, P, knum), dtype=torch.float32, device=dev)
    w0 = torch.empty((B, P, knum), dtype=torch.float32, device=dev)
    w1 = torch.empty((B, P, knum), dtype=torch.float32, device=dev)
    ws = _lib.scratch(_lib.lib().dibr_b200_deftet_workspace_bytes(B, F), dev)
    _lib.call("dibr_b200_deftet_sparse_render_forward", dev,
              B, F, P, int(knum), face_vertices_z, face_vertices_image, face_bboxes,
              pixel_coords, pixel_depth_ranges, float(eps), idx, depth, w0, w1,
              ws, ws.numel(), what=fn)
    return [idx, depth, w0, w1]


@_fp64_via_fp32
def deftet_sparse_render_backward_cuda(grad_interpolated_features, face_idx, weights, face_vertices_image,
                                       face_features, eps):
    """deftet.cpp:115-170 -> [grad_face_vertices_image, grad_face_features]."""
    fn = "deftet_sparse_render_backward_cuda"
    dev = _check_all(fn, [("grad_interpolated_features", grad_interpolated_features), ("face_idx", face_idx),
                          ("weights", weights), ("face_vertices_image", face_vertices_image),
                          ("face_features", face_features)])
    B, P, K, D = grad_interpolated_features.shape
    F = face_vertices_image.shape[1]
    _check_size(fn, "face_idx", face_idx, (B, P, K))
    _check_size(fn, "weights", weights, (B, P, K, 3))
    _check_size(fn, "face_vertices_image", face_vertices_image, (B, F, 3, 2))
    _check_size(fn, "face_features", face_features, (B, F, 3, D))
    g_xy = torch.empty_like(face_vertices_image)
    g_ff = torch.empty_like(face_features)
    _lib.call("dibr_b200_deftet_sparse_render_backward", dev,
              B, F, P, K, D, grad_interpolated_features, face_idx, weights,
              face_vertices_image, face_features, float(eps), g_xy, g_ff, what=fn)
    return [g_xy, g_ff]


def _check_sg(fn, named):
    """unbatched_reduced_sg_inner_product.cpp:57-103: same GPU, contiguous, same type, sizes."""
    dev = _check_all(fn, named)
    dtypes = {t.dtype for _, t in named}
    if len(dtypes) > 1:
        raise RuntimeError(f"{fn}: expected all tensors to have the same type, got {sorted(map(str, dtypes))}")
    t = dict(named)
    num_sg, num_other = t["intensity"].shape[0], t["other_intensity"].shape[0]
    for name, shape in (("grad_out", (num_sg, 3)), ("intensity", (num_sg, 3)), ("direction", (num_sg, 3)),
                        ("sharpness", (num_sg,)), ("other_intensity", (num_other, 3)),
                        ("other_direction", (num_other, 3)), ("other_sharpness", (num_other,))):
        if name in t:
            _check_size(fn, name, t[name], shape)
    return dev


def unbatched_reduced_sg_inner_product_forward_cuda(intensity, direction, sharpness,
                                                    other_intensity, other_direction, other_sharpness):
    """unbatched_reduced_sg_inner_product.cpp:49-123 -> output (num_sg, 3)."""
    from .render.lighting import sg
    args = [("intensity", intensity), ("direction", direction), ("sharpness", sharpness),
            ("other_intensity", other_intensity), ("other_direction", other_direction),
            ("other_sharpness", other_sharpness)]
    _check_sg("unbatched_reduced_sg_inner_product_forward_cuda", args)
    return sg.forward_sg_inner_product(*[t for _, t in args])


def unbatched_reduced_sg_inner_product_backward_cuda(grad_out, intensity, direction, sharpness,
                                                     other_intensity, other_direction, other_sharpness):
    """unbatched_reduced_sg_inner_product.cpp:125-218 -> [grad_intensity, grad_direction, grad_sharpness,
    grad_other_intensity, grad_other_direction, grad_other_sharpness]."""
    from .render.lighting import sg
    args = [("grad_out", grad_out), ("intensity", intensity), ("direction", direction), ("sharpness", sharpness),
            ("other_intensity", other_intensity), ("other_direction", other_direction),
            ("other_sharpness", other_sharpness)]
    _check_sg("unbatched_reduced_sg_inner_product_backward_cuda", args)
    return sg.backward_sg_inner_product(*[t for _, t in args])


def unbatched_mesh_intersection_cuda(points, verts_1, verts_2, verts_3):
    """mesh_intersection.cpp:32-65 -> counts (num_points,) of the points' type: for each point, the faces
    (verts_1[f], verts_2[f], verts_3[f]) its +x ray crosses, as the reference's kernel counts them
    (check_sign's corners, gathered and normalised by the caller).  float32 or float64."""
    fn = "unbatched_mesh_intersection_cuda"
    named = [("points", points), ("verts_1", verts_1), ("verts_2", verts_2), ("verts_3", verts_3)]
    dev = _check_all(fn, named, float_dtype=points.dtype)
    if len({t.dtype for _, t in named}) > 1:
        raise RuntimeError(f"{fn}: expected all tensors to have the same type, "
                           f"got {[str(t.dtype) for _, t in named]}")
    num_points, num_faces = points.shape[0], verts_1.shape[0]
    _check_size(fn, "points", points, (num_points, 3))
    for name, t in named[1:]:
        _check_size(fn, name, t, (num_faces, 3))
    dtype = {torch.float32: _lib.DTYPE_F32, torch.float64: _lib.DTYPE_F64}.get(points.dtype)
    if dtype is None:
        raise RuntimeError(f"{fn} not implemented for '{str(points.dtype).replace('torch.', '')}'")
    out = torch.empty((num_points,), dtype=points.dtype, device=dev)
    build, query = _lib.check_sign_workspace_bytes(1, num_faces, num_points, dtype, fn)
    ws = _lib.scratch(build + query, dev)
    _lib.call("dibr_b200_mesh_intersection_count", dev, num_faces, num_points, dtype, points, verts_1, verts_2,
              verts_3, out, ws, ws.numel(), what=fn)
    return out


def unbatched_mcube_forward_cuda(voxelgrid, iso_value):
    """unbatched_mcube.cpp -> [vertices (nv, 3) float32, faces (nf, 3) int32]: marching cubes on one
    already-padded grid (X, Y, Z) float32, as ``voxelgrids_to_trianglemeshes`` calls it per view."""
    from .ops.conversions.voxelgrid import unbatched_mcube_forward
    return unbatched_mcube_forward(voxelgrid, iso_value)


def _check_triangle_distance(fn, named, sizes):
    """CHECK_CUDA, then CHECK_CONTIGUOUS, then CHECK_SIZES (unbatched_triangle_distance.cpp), in its order."""
    for name, t in named:
        if not t.is_cuda:
            raise RuntimeError(f"{name} must be a CUDA tensor")
    for name, t in named:
        if not t.is_contiguous():
            raise RuntimeError(f"{name} must be contiguous")
    for name, t in named:
        if tuple(t.shape) != tuple(sizes[name]):
            raise RuntimeError(f"{name} must of size {{{', '.join(str(s) for s in sizes[name])}}}")
    dev = named[0][1].device
    for name, t in named:
        if t.device != dev:
            raise RuntimeError(f"{fn}: expected all tensors on one device; {name} is on {t.device}")


def _check_types(fn, named):
    for name, t, dtype in named:
        if t.dtype != dtype:
            raise RuntimeError(f"{fn}: expected {name} of type {dtype}, got {t.dtype}")


def unbatched_triangle_distance_forward_cuda(points, face_vertices, dist, face_idx, dist_type):
    """unbatched_triangle_distance.cpp:43-72: points (N, 3), face_vertices (F, 3, 3) -> written into
    dist (N), face_idx (N) int64 and dist_type (N) int32; float32 or float64.  With F = 0 the outputs are
    left as they are, as in the reference."""
    from .metrics.trianglemesh import _dtype_flag, _pmd_forward
    fn = "unbatched_triangle_distance_forward_cuda"
    named = [("points", points), ("face_vertices", face_vertices), ("dist", dist), ("face_idx", face_idx),
             ("dist_type", dist_type)]
    N, F = points.shape[0], face_vertices.shape[0]
    _check_triangle_distance(fn, named, {"points": (N, 3), "face_vertices": (F, 3, 3), "dist": (N,),
                                         "face_idx": (N,), "dist_type": (N,)})
    _dtype_flag(fn, points.dtype)
    _check_types(fn, [("face_vertices", face_vertices, points.dtype), ("dist", dist, points.dtype),
                      ("face_idx", face_idx, torch.int64), ("dist_type", dist_type, torch.int32)])
    with torch.cuda.device(points.device):
        _pmd_forward(points[None], face_vertices[None], dist, face_idx, dist_type)


def unbatched_triangle_distance_backward_cuda(grad_dist, points, face_vertices, face_idx, dist_type, grad_points,
                                              grad_face_vertices):
    """unbatched_triangle_distance.cpp:74-114: grad_points (N, 3) written, grad_face_vertices (F, 3, 3)
    added to, in ascending point order per face (no float atomics)."""
    from .metrics.trianglemesh import _dtype_flag, _pmd_backward
    fn = "unbatched_triangle_distance_backward_cuda"
    named = [("grad_dist", grad_dist), ("points", points), ("face_vertices", face_vertices), ("face_idx", face_idx),
             ("dist_type", dist_type), ("grad_points", grad_points), ("grad_face_vertices", grad_face_vertices)]
    N, F = points.shape[0], face_vertices.shape[0]
    _check_triangle_distance(fn, named, {"grad_dist": (N,), "points": (N, 3), "face_vertices": (F, 3, 3),
                                         "face_idx": (N,), "dist_type": (N,), "grad_points": (N, 3),
                                         "grad_face_vertices": (F, 3, 3)})
    _dtype_flag(fn, points.dtype)
    _check_types(fn, [("grad_dist", grad_dist, points.dtype), ("face_vertices", face_vertices, points.dtype),
                      ("face_idx", face_idx, torch.int64), ("dist_type", dist_type, torch.int32),
                      ("grad_points", grad_points, points.dtype),
                      ("grad_face_vertices", grad_face_vertices, points.dtype)])
    with torch.cuda.device(points.device):
        _pmd_backward(grad_dist[None], points[None], face_vertices[None], face_idx, dist_type, grad_points,
                      grad_face_vertices)


# kaolin._C.metrics.<op>, as bindings.cpp lays it out
metrics = types.SimpleNamespace(
    unbatched_triangle_distance_forward_cuda=unbatched_triangle_distance_forward_cuda,
    unbatched_triangle_distance_backward_cuda=unbatched_triangle_distance_backward_cuda,
)

# kaolin._C.ops.{mesh,conversions}.<op>, as bindings.cpp lays them out
ops = types.SimpleNamespace(mesh=types.SimpleNamespace(
    unbatched_mesh_intersection_cuda=unbatched_mesh_intersection_cuda,
), conversions=types.SimpleNamespace(
    unbatched_mcube_forward_cuda=unbatched_mcube_forward_cuda,
))

# kaolin._C.render.{mesh,sg}.<op> namespaces, as bindings.cpp:42,111-115,129-133 lays them out
render = types.SimpleNamespace(sg=types.SimpleNamespace(
    unbatched_reduced_sg_inner_product_forward_cuda=unbatched_reduced_sg_inner_product_forward_cuda,
    unbatched_reduced_sg_inner_product_backward_cuda=unbatched_reduced_sg_inner_product_backward_cuda,
), mesh=types.SimpleNamespace(
    packed_rasterize_forward_cuda=packed_rasterize_forward_cuda,
    rasterize_backward_cuda=rasterize_backward_cuda,
    dibr_soft_mask_forward_cuda=dibr_soft_mask_forward_cuda,
    dibr_soft_mask_backward_cuda=dibr_soft_mask_backward_cuda,
    deftet_sparse_render_forward_cuda=deftet_sparse_render_forward_cuda,
    deftet_sparse_render_backward_cuda=deftet_sparse_render_backward_cuda,
))
