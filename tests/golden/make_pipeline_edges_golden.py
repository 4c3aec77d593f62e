"""Regenerates tests/golden/pipeline_edges.npz from the reference (run in the build container only).

    python tests/golden/make_pipeline_edges_golden.py

float64 CPU outputs and autograd gradients of the reference's OWN functions, imported in place, on
the edge scenes of tests/test_pipeline_edges_{cpu,gpu}.py.  They pin the float64 run of
oracle/pipeline.py's torch restatements, which is the judge of the GPU tests:
  dg_*  prepare_vertices on a mesh with zero-area faces ((a,a,b), (a,a,a), three collinear vertices)
        under cameras whose arithmetic is exact, so that collinear stays collinear
  ep_*  prepare_vertices on a scene scaled, camera distance included, so that the length of the
        un-normalised normal spans 1e-13 .. 1e-7: the range where its 1e-10 matters
  tk_*  texture_mapping on every pair of the clamp / border kink coordinates, 5x1 and 4x8 textures
  mi_*  mask_iou on empty, full, complementary and out-of-range masks
"""
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))
from oracle import ref_import  # noqa: E402

utils = ref_import.module("kaolin.render.mesh.utils")
metrics = ref_import.module("kaolin.metrics.render")

out = {}
g = torch.Generator().manual_seed(20261016)
D = torch.float64
rand = lambda *s: torch.rand(s, generator=g, dtype=torch.float32)     # inputs are float32 values


def run_prepare(tag, vertices, faces, proj, rot, trans, transform):
    """Both camera conventions on float64 copies of float32 inputs; stores inputs, outputs, gradients."""
    B, F = vertices.shape[0], faces.shape[0]
    w = [rand(B, F, 3, 3), rand(B, F, 3, 2), rand(B, F, 3)]
    out.update({f"{tag}_vertices": vertices.numpy(), f"{tag}_faces": faces.numpy(), f"{tag}_proj": proj.numpy(),
                f"{tag}_rot": rot.numpy(), f"{tag}_trans": trans.numpy(), f"{tag}_transform": transform.numpy(),
                f"{tag}_w1": w[0].numpy(), f"{tag}_w2": w[1].numpy(), f"{tag}_w3": w[2].numpy()})
    for mode in ("T", "Rt"):
        v = vertices.to(D).requires_grad_(True)
        if mode == "T":
            cam = dict(camera_transform=transform.to(D).requires_grad_(True))
        else:
            cam = dict(camera_rot=rot.to(D).requires_grad_(True), camera_trans=trans.to(D).requires_grad_(True))
        res = utils.prepare_vertices(v, faces, proj.to(D), **cam)
        sum((o * wi.to(D)).sum() for o, wi in zip(res, w)).backward()
        for name, o in zip(("fvc", "fvi", "fn"), res):
            out[f"{tag}_{mode}_{name}"] = o.detach().numpy()
        out[f"{tag}_{mode}_g_vertices"] = v.grad.numpy()
        for name, t in cam.items():
            out[f"{tag}_{mode}_g_{name[7:]}"] = t.grad.numpy()


def look_at(pos):
    """(B,3) camera positions looking at the origin -> rotation (B,3,3) rows x, y, z and translation."""
    z = pos / pos.norm(dim=1, keepdim=True)
    x = torch.linalg.cross(torch.tensor([[0., 1., 0.]]).expand_as(z), z)
    x = x / x.norm(dim=1, keepdim=True)
    y = torch.linalg.cross(z, x)
    return torch.stack([x, y, z], dim=1), pos.clone()


def transform_of(rot, trans):
    """The (B,4,3) matrix of the same camera: [p, 1] @ T == (p - t) @ R^T."""
    rt = rot.transpose(1, 2)
    return torch.cat([rt, -(trans.view(-1, 1, 3) @ rt)], dim=1)


proj = torch.tensor([[1 / math.tan(math.pi / 8)], [1 / math.tan(math.pi / 8)], [-1.]], dtype=torch.float32)

# ---- dg: zero-area faces.  Vertices on a 1/64 lattice, signed axis permutations as rotations and
# power-of-two translations: every camera-space coordinate is exact in float32 AND float64, so the
# collinear triple stays collinear and its cross product is exactly zero on both sides.
verts = (torch.randint(-32, 33, (2, 12, 3), generator=g).float() / 64)
verts[:, 8] = torch.tensor([0.25, 0.5, -0.25]); verts[:, 9] = torch.tensor([0.5, 0.25, 0.])
verts[:, 10] = torch.tensor([0.75, 0., 0.25])                 # 8, 9, 10 collinear
faces = torch.tensor([[0, 1, 2], [3, 3, 4], [2, 3, 4], [5, 5, 5], [4, 5, 6], [8, 9, 10], [6, 7, 0],
                      [10, 8, 9], [1, 3, 5], [11, 0, 11], [7, 2, 4], [0, 2, 6]])
rot = torch.tensor([[[1., 0., 0.], [0., 1., 0.], [0., 0., 1.]],
                    [[0., 0., -1.], [0., 1., 0.], [1., 0., 0.]]])
trans = torch.tensor([[0.5, -0.25, 4.], [4., 0.125, 0.5]])
run_prepare("dg", verts, faces, proj, rot, trans, transform_of(rot, trans))
out["dg_degenerate"] = np.array([1, 3, 5, 7, 9])

# ---- ep: one random mesh seen by 4 cameras, view b scaled as a whole by s_b (vertices AND camera
# position): edges ~ s, camera-space coordinates ~ 3 s, so the cross product keeps its float32
# conditioning while its length L ~ s^2 runs through 1e-13 .. 1e-7 either side of the 1e-10.
scales = torch.tensor([7e-7, 9e-6, 1.1e-4, 1.3e-3])
base = rand(1, 24, 3) - 0.5
faces = torch.stack([torch.randperm(24, generator=g)[:3] for _ in range(40)]).long()
ang = torch.tensor([0.3, 1.9, 3.6, 5.2])
rot, pos = look_at(torch.stack([3 * torch.cos(ang), torch.tensor([0.4, -0.7, 0.1, 0.9]), 3 * torch.sin(ang)], dim=1))
verts = base * scales.view(4, 1, 1)
trans = pos * scales.view(4, 1)
run_prepare("ep", verts, faces, proj, rot, trans, transform_of(rot, trans))


# ---- tk: every pair of kink coordinates.  h = half a texel of an axis of `size` texels.
def kinks(size):
    h = np.float32(0.5 / size)
    one = np.float32(1)
    up = lambda x: np.nextafter(np.float32(x), np.float32(np.inf))
    dn = lambda x: np.nextafter(np.float32(x), np.float32(-np.inf))
    d = np.float32(2.0 ** -24)      # the step of 2u - 1 near +-1: what the grid coordinate resolves
    vals = [-1., -0., 0., 1e-40, dn(h), h, up(h), h - d, h + d, dn(one - h), one - h, up(one - h),
            one - h - d, one - h + d, 0.5, 0.3, one - d, 1., 1. + 2.0 ** -23, 2., np.inf, -np.inf]
    return np.array(vals, np.float32)


for tag, (Ht, Wt) in (("tk51", (5, 1)), ("tk48", (4, 8))):
    ku, kv = kinks(Wt), kinks(Ht)
    uv = torch.from_numpy(np.stack(np.meshgrid(ku, kv, indexing="ij"), -1).reshape(1, -1, 2)).repeat(2, 1, 1)
    tex = rand(2, 3, Ht, Wt)
    gw = rand(2, uv.shape[1], 3)
    out.update({f"{tag}_uv": uv.numpy(), f"{tag}_tex": tex.numpy(), f"{tag}_gw": gw.numpy()})
    for mode in ("nearest", "bilinear"):
        u, t = uv.to(D).requires_grad_(True), tex.to(D).requires_grad_(True)
        o = utils.texture_mapping(u, t, mode=mode)
        (o * gw.to(D)).sum().backward()
        out[f"{tag}_{mode}_out"] = o.detach().numpy()
        out[f"{tag}_{mode}_g_tex"] = t.grad.numpy()
        out[f"{tag}_{mode}_g_uv"] = (u.grad if u.grad is not None else torch.zeros_like(u)).numpy()

# ---- mi: mask values at the edges of the loss
r = (rand(3, 4, 5) > 0.5).float()
full, empty = torch.ones(3, 4, 5), torch.zeros(3, 4, 5)
one_empty = full.clone(); one_empty[1] = 0
cases = {"empty": (empty, empty), "full": (full, full), "one_empty": (one_empty, one_empty),
         "complement": (1 - r, r), "range": (rand(3, 4, 5) * 4 - 2, rand(3, 4, 5) * 3 - 1)}
for name, (a, b) in cases.items():
    l, rr = a.to(D).requires_grad_(True), b.to(D).requires_grad_(True)
    loss = metrics.mask_iou(l, rr)
    (loss * 1.7).backward()
    out.update({f"mi_{name}_lhs": a.numpy(), f"mi_{name}_rhs": b.numpy(), f"mi_{name}_loss": np.float64(loss.item()),
                f"mi_{name}_g_lhs": l.grad.numpy(), f"mi_{name}_g_rhs": rr.grad.numpy()})
out["mi_gscale"] = np.float64(1.7)

np.savez_compressed(os.path.join(HERE, "pipeline_edges.npz"), **out)
print("wrote", os.path.join(HERE, "pipeline_edges.npz"), len(out), "arrays")
