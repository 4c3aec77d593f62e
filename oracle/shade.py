"""TEST INFRASTRUCTURE — sg_shade of kaolin/render/easy_render/mesh.py:427-464 restated in torch:
boolean gathers of the covered pixels, the normal normalised, the pinhole view ray of every pixel of the
custom-resolution grid (kaolin/render/camera/raygen.py), the diffuse term of oracle/lighting.py and the
specular term of oracle/specular.py, scattered back into zero images.  float64 inputs give the tests'
reference.  Never imported by kaolin_b200.

The camera is plain arrays: R (B,3,3) world to camera, x0, y0, focal_x, focal_y (B,), and the camera
image size (width, height)."""
import torch

from . import lighting as OL
from . import specular as OS


def view_dirs(R, x0, y0, focal_x, focal_y, width, height, H, W):
    """(B,H,W,3): minus the unit pinhole ray through the centre of each pixel of an H x W grid spread
    over the width x height image plane (pixel (i, j) at ((j + 1/2) width / W, (i + 1/2) height / H))."""
    dt = R.dtype
    sx, sy = width / W, height / H
    # the grid is float32, as the reference's, and takes the camera's dtype after the scaling
    px = (sx * torch.arange(W, dtype=torch.float32) + sx / 2.).to(dt)
    py = (sy * torch.arange(H, dtype=torch.float32) + sy / 2.).to(dt)
    px = px[None, None, :] - x0[:, None, None]
    py = py[None, :, None] + y0[:, None, None]
    nx = 2 * (px / width) - 1.
    ny = 2 * (py / height) - 1.
    tan_x = (width / 2.) / focal_x
    tan_y = (height / 2.) / focal_y
    B = R.shape[0]
    d = torch.stack(torch.broadcast_tensors(nx * tan_x[:, None, None], -ny * tan_y[:, None, None],
                                            -torch.ones((B, H, W), dtype=dt)), dim=-1)
    w = torch.einsum('bki,bhwk->bhwi', R, d)          # R^T d
    return -(w / torch.linalg.norm(w, dim=-1, keepdim=True))


def sg_shade(view, face_idx, albedo, spec_albedo, roughness, normals, amp, dirs, sharp):
    """(diffuse, specular, img), each (B,H,W,3), of a G-buffer with per-pixel ``view`` (B,H,W,3)."""
    mask = face_idx >= 0
    n = torch.nn.functional.normalize(normals[mask], dim=-1)
    d = OL.sg_diffuse_inner_product(amp, dirs, sharp, n, albedo[mask])
    s = OS.sg_warp_specular_term(amp, dirs, sharp, n, roughness.reshape(mask.shape)[mask], view[mask],
                                 spec_albedo[mask])
    zeros = normals.new_zeros(normals.shape[:3] + (3,))
    diffuse = zeros.index_put((mask,), d)
    specular = zeros.index_put((mask,), s)
    return diffuse, specular, zeros.index_put((mask,), d + s)
