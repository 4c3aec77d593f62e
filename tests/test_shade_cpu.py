"""sg_shade, texture_sample_materials and render_mesh without a GPU: the reference's signatures, the
C ABI's host-side argument checks, no CPU fallback, the camera-gradient refusal, and the fp64
restatement (oracle/shade.py) against the reference's own goldens (tests/golden/shade.npz)."""
import ctypes
import inspect
import os
import types

import numpy as np
import pytest
import torch

from kaolin_b200 import _lib
from kaolin_b200.render import easy_render
from oracle import ref_import
from oracle import shade as OSH

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "shade.npz"))
LIGHTS = (1, 2, 7, 8, 40)


class Cam(types.SimpleNamespace):
    def __len__(self):
        return self.extrinsics.R.shape[0]


def make_camera(device="cpu", requires_grad=False):
    """A duck-typed camera from the golden's arrays."""
    t = lambda k: torch.from_numpy(G[k]).float().to(device).requires_grad_(requires_grad)
    return Cam(extrinsics=types.SimpleNamespace(R=t("cam_R")), x0=t("cam_x0"), y0=t("cam_y0"),
               focal_x=t("cam_focal_x"), focal_y=t("cam_focal_y"), width=int(G["cam_width"]),
               height=int(G["cam_height"]))


def inputs(L, device="cpu", dtype=torch.float32):
    t = lambda k: torch.from_numpy(G[f"L{L}_{k}"]).to(device, dtype)
    face_idx = torch.from_numpy(G[f"L{L}_face_idx"]).to(device)
    return [face_idx] + [t(k) for k in ("albedo", "spec_albedo", "roughness", "normals", "amp", "dir", "sharp")]


@pytest.mark.skipif(not ref_import.available(), reason="needs the reference's sources")
def test_signatures_match_the_reference():
    ref = ref_import.module("kaolin.render.easy_render.mesh")
    for name in ("sg_shade", "render_mesh", "texture_sample_materials"):
        ours, theirs = (inspect.signature(getattr(m, name)).parameters for m in (easy_render, ref))
        assert [(p.name, p.default) for p in ours.values()] == [(p.name, p.default) for p in theirs.values()], name
    assert [p.name for p in easy_render.RenderPass] == [p.name for p in ref.RenderPass]


def test_abi_rejects_bad_arguments_on_the_host():
    lib = _lib.lib()
    assert lib.dibr_b200_sg_shade_workspace_bytes(-1) == 0
    assert lib.dibr_b200_sg_shade_workspace_bytes(1) == lib.dibr_b200_specular_workspace_bytes(1)
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    fwd = lambda B, H, W, L, cam=p, face=p, out=p: lib.dibr_b200_sg_shade_forward(
        B, H, W, L, cam, face, p, p, p, p, p, p, p, out, out, out, None)
    assert fwd(-1, 4, 4, 1) == _lib.EINVAL
    assert fwd(1, 4, 4, -1) == _lib.EINVAL
    assert fwd(1, 16385, 4, 1) == _lib.ESIZE
    assert fwd(1, 4, 16385, 1) == _lib.ESIZE
    assert fwd(1, 4, 4, 1, cam=None) == _lib.EINVAL
    assert fwd(1, 4, 4, 1, face=None) == _lib.EINVAL
    assert fwd(1, 4, 4, 1, out=None) == _lib.EINVAL
    assert fwd(0, 4, 4, 0, cam=None, face=None, out=None) == 0          # nothing to do, nothing launched
    bwd = lambda L, ws, nbytes: lib.dibr_b200_sg_shade_backward(
        1, 4, 4, L, p, p, p, p, p, p, p, p, p, p, p, p, None, None, None, None, p, None, None, ws, nbytes, None)
    assert bwd(1, None, 1 << 20) == _lib.EINVAL                        # light gradients need a workspace
    assert bwd(1, p, 16) == _lib.EWORKSPACE
    assert lib.dibr_b200_sg_shade_backward(1, 4, 4, 1, p, None, p, p, p, p, p, p, p, p, p, p, p, p, p, p,
                                           None, None, None, None, 0, None) == _lib.EINVAL


def test_cpu_tensors_raise():
    with pytest.raises(RuntimeError, match="CUDA"):
        easy_render.sg_shade(make_camera(), *inputs(1))
    with pytest.raises(RuntimeError):
        easy_render.sg_shade(make_camera(), *inputs(1, dtype=torch.float64))


def test_camera_requiring_grad_raises():
    with pytest.raises(NotImplementedError, match="camera"):
        easy_render.sg_shade(make_camera(requires_grad=True), *inputs(1))
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA"):    # no gradient asked: on to the checks
        easy_render.sg_shade(make_camera(requires_grad=True), *inputs(1))


def test_nvdiffrast_backend_raises():
    with pytest.raises(ValueError, match="nvdiffrast"):
        easy_render.texture_sample_materials('nvdiffrast', torch.zeros((1, 2, 2), dtype=torch.long), None)


def oracle_view(dtype=torch.float64):
    t = lambda k: torch.from_numpy(G[k]).to(dtype)
    return OSH.view_dirs(t("cam_R"), t("cam_x0"), t("cam_y0"), t("cam_focal_x"), t("cam_focal_y"),
                         int(G["cam_width"]), int(G["cam_height"]), *G["L1_face_idx"].shape[1:])


def test_oracle_view_matches_the_reference_rays():
    v = oracle_view()
    ref = torch.from_numpy(G["view"])
    assert float((v - ref).abs().max()) <= 1e-12


@pytest.mark.parametrize("L", LIGHTS)
def test_oracle_reproduces_the_goldens(L):
    face_idx, *rest = inputs(L, dtype=torch.float64)
    leaves = [t.clone().requires_grad_(True) for t in rest]
    outs = OSH.sg_shade(oracle_view(), face_idx, *leaves)
    sum((o * torch.from_numpy(G[f"L{L}_w_{n}"])).sum() for o, n in zip(outs, ("diffuse", "specular", "img"))).backward()
    for o, n in zip(outs, ("diffuse", "specular", "img")):
        ref = torch.from_numpy(G[f"L{L}_{n}"])
        assert float((o.detach() - ref).abs().max()) <= 1e-5 * float(ref.abs().max()), n
    for t, k in zip(leaves, ("albedo", "spec_albedo", "roughness", "normals", "amp", "dir", "sharp")):
        ref = torch.from_numpy(G[f"L{L}_g_{k}"])
        assert float((t.grad - ref).abs().max()) <= 1e-5 * float(ref.abs().max()), k
