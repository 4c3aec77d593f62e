"""The seven kernels of kaolin_b200/csrc/mesh_pipeline.cu (prepare_vertices, texture_mapping, mask_iou)
at the inputs where they can be wrong: the scale where the normal's 1e-10 matters, zero-area faces,
one vertex in 100 000 faces, texel boundaries and centres, the clamp and border kinks of the
coordinate gradient, 2^20 samples on one texel, launch-geometry edges of the mask sums, inputs of the
wrong element type or alignment.

The judge is oracle/pipeline.py's torch restatements run in float64 on the CPU (pinned to the
reference by tests/test_pipeline_edges_cpu.py) on the float32 inputs the kernel got, plus, for which
texel a coordinate selects, torch's own CUDA ``grid_sample`` in float32: the library path the reference
takes.  Every comparison is per element, ``|a - ref| <= bound`` with the bound derived from the
operation and computed on the float64 side; discrete results (which texel, which entries are exactly
zero, NaN / inf patterns) are compared exactly."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import pipeline as P
from kaolin_b200 import _lib
from kaolin_b200.metrics.render import mask_iou
from kaolin_b200.render.mesh import prepare_vertices, texture_mapping

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 2.0 ** -24         # unit roundoff of float32
D = torch.float64
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "pipeline_edges.npz"))
MODES = ["nearest", "bilinear"]


def f64(t):
    return t.detach().to("cpu", D)


def dev(t, grad=False):
    return t.detach().to(DEV, torch.float32).requires_grad_(grad)


def within(a, ref, bound, what):
    """Per element: NaN and inf where the float64 side has them, else |a - ref| <= bound."""
    a = f64(a)
    assert a.shape == ref.shape, (what, a.shape, ref.shape)
    fin = torch.isfinite(ref)
    assert torch.equal(torch.isnan(a), torch.isnan(ref)), f"{what}: NaN pattern"
    assert torch.equal(a[torch.isinf(ref)], ref[torch.isinf(ref)]), f"{what}: inf pattern"
    err = torch.where(fin, (a - ref).abs(), torch.zeros_like(ref))
    bound = torch.as_tensor(bound, dtype=D).expand_as(ref)
    bad = fin & ~(err <= bound)
    if bad.any():
        i = int(torch.where(bad, err / bound.clamp_min(1e-300), torch.zeros_like(err)).argmax())
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside their bound; worst: "
                             f"got {a.reshape(-1)[i].item()!r}, float64 {ref.reshape(-1)[i].item()!r}, "
                             f"bound {bound.reshape(-1)[i].item():.3e}")


def scatter_k(n):
    """A float32 sum of n terms accumulated one at a time in any order (atomics): each addition rounds
    the running sum by at most EPS * |partial sum| <= EPS * sum|terms|; n such errors add up like a
    random walk, ~ sqrt(n), and 4 sqrt(n) + 8 leaves room for its tail.  Times EPS * sum|terms|."""
    return 4 * math.sqrt(max(n, 1)) + 8


# =================================================================================================
# prepare_vertices
def look_at(pos):
    z = pos / pos.norm(dim=1, keepdim=True)
    x = torch.linalg.cross(torch.tensor([[0., 1., 0.]]).expand_as(z), z)
    x = x / x.norm(dim=1, keepdim=True)
    return torch.stack([x, torch.linalg.cross(z, x), z], dim=1), pos.clone()


def transform_of(rot, trans):
    rt = rot.transpose(1, 2)
    return torch.cat([rt, -(trans.view(-1, 1, 3) @ rt)], dim=1)


PROJ = torch.tensor([[1 / math.tan(math.pi / 8)], [1 / math.tan(math.pi / 8)], [-1.]])


def cameras(B, seed, dist=3.0):
    g = torch.Generator().manual_seed(seed)
    ang = torch.rand(B, generator=g) * 2 * math.pi
    pos = torch.stack([dist * torch.cos(ang), torch.rand(B, generator=g) * 2 - 1, dist * torch.sin(ang)], dim=1)
    return look_at(pos)


def abscross(a, b):
    """|cross(a, b)| bounded term by term, for non-negative a, b."""
    return torch.stack([a[..., 1] * b[..., 2] + a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] + a[..., 0] * b[..., 2],
                        a[..., 0] * b[..., 1] + a[..., 1] * b[..., 0]], dim=-1)


class PV:
    """float64 results of prepare_vertices on float32 inputs, with the per-element float32 error bounds."""

    def __init__(self, v, faces, mode, rot, trans, transform, w, proj=PROJ):
        self.mode = mode
        v64, proj64 = f64(v).requires_grad_(True), f64(proj)
        self.cam = ({"camera_transform": f64(transform).requires_grad_(True)} if mode == "T" else
                    {"camera_rot": f64(rot).requires_grad_(True), "camera_trans": f64(trans).requires_grad_(True)})
        faces = faces.cpu()
        B, V, F = v64.shape[0], v64.shape[1], faces.shape[0]
        self.out = P.prepare_vertices_torch(v64, faces, proj64, **self.cam)
        if w is not None:
            sum((o * f64(wi)).sum() for o, wi in zip(self.out, w) if wi is not None).backward()
        self.g_v = v64.grad if v64.grad is not None else torch.zeros_like(v64)
        self.g_cam = {k: (t.grad if t.grad is not None else torch.zeros_like(t)) for k, t in self.cam.items()}
        fvc, fvi, fn = (o.detach() for o in self.out)
        va = v64.detach().abs()
        # camera-space vertex: a 3- or 4-term dot product by fused multiply-adds, each rounding at most
        # EPS * (sum of |terms|); in Rt mode p - t rounds first, by EPS * (|p| + |t|) at most
        if mode == "T":
            Ta = self.cam["camera_transform"].detach().abs()
            dvc = 4 * EPS * (va @ Ta[:, :3] + Ta[:, 3:])
            self.lin = self.cam["camera_transform"].detach()[:, :3].transpose(1, 2)       # g_v = g_vc @ lin
        else:
            Ra, ta = self.cam["camera_rot"].detach().abs(), self.cam["camera_trans"].detach().abs().view(B, 1, 3)
            dvc = 5 * EPS * ((va + ta) @ Ra.transpose(1, 2))
            self.lin = self.cam["camera_rot"].detach()
        dfv = dvc[:, faces]                                        # (B,F,3,3)
        self.b_fvc = dfv
        # image point x px / (z pz): two products and a correctly rounded division (3 EPS relative),
        # plus the numerator's and the denominator's own errors carried through the quotient
        z = fvc[..., 2:3].abs()
        self.b_fvi = dfv[..., :2] / z * (proj64[:2, 0] / proj64[2, 0]).abs() + fvi.abs() * (dfv[..., 2:3] / z + 4 * EPS)
        # normal c / (L + 1e-10), c = e0 x e1: an edge is a difference of two vertices (their errors add,
        # plus one rounding); each component of c is two products and a difference
        e0, e1 = fvc[:, :, 1] - fvc[:, :, 0], fvc[:, :, 2] - fvc[:, :, 0]
        de0 = dfv[:, :, 1] + dfv[:, :, 0] + EPS * e0.abs()
        de1 = dfv[:, :, 2] + dfv[:, :, 0] + EPS * e1.abs()
        c = torch.linalg.cross(e0, e1)
        dc = abscross(e0.abs(), de1) + abscross(de0, e1.abs()) + 3 * EPS * abscross(e0.abs(), e1.abs())
        self.L = c.norm(dim=-1, keepdim=True)
        Le = self.L + 1e-10
        dL = dc.norm(dim=-1, keepdim=True) + 3 * EPS * self.L
        # the 1e-10 is a float32 constant in the kernel: 1.3e-8 relative off the double one, under EPS
        self.b_fn = dc / Le + fn.abs() * (dL / Le + 4 * EPS)
        if w is None:
            return
        # gradients.  G: the float64 gradient wrt each face corner in camera space.  The kernel forms it from
        # c and 1 / L, so it inherits their relative error |dc| / L (bounded above), a few times over as L enters
        # squared: 16 EPS + 4 |dc| / L of the face's largest entry.  For a zero-area face the normal gradient is
        # g_n / 1e-10 crossed with an edge, and inherits the edge's relative error instead.  Corners are summed per
        # vertex by atomics (scatter_k), then a (3,3) product takes the camera-space gradient to the inputs.
        fv = fvc.clone().requires_grad_(True)
        vi = fv[..., :2] * proj64[:2, 0] / (fv[..., 2:3] * proj64[2, 0])
        n = torch.linalg.cross(fv[:, :, 1] - fv[:, :, 0], fv[:, :, 2] - fv[:, :, 0])
        n = n / (n.norm(dim=2, keepdim=True) + 1e-10)
        sum((o * f64(wi)).sum() for o, wi in zip((fv, vi, n), w) if wi is not None).backward()
        Gc = fv.grad                                                # (B,F,3,3)
        emax = torch.maximum(e0.abs().amax(-1), e1.abs().amax(-1))
        L1 = self.L[..., 0]
        rel = torch.where(L1 > 0, dc.norm(dim=-1) / L1.clamp_min(1e-300),
                          torch.maximum(de0.amax(-1), de1.amax(-1)) / emax.clamp_min(1e-300))
        rel = 16 * EPS + 4 * torch.where((L1 == 0) & (emax == 0), torch.zeros_like(rel), rel)
        b_corner = (rel * Gc.abs().amax(dim=(2, 3)))[..., None, None].expand_as(Gc)
        idx = faces.reshape(-1)
        deg = int(torch.bincount(idx, minlength=V).max()) if F else 0
        gather = lambda x: torch.zeros((B, V, 3), dtype=D).index_add_(1, idx, x.reshape(B, F * 3, 3))
        self.g_vc = gather(Gc)
        self.b_gvc = gather(b_corner) + scatter_k(deg) * EPS * gather(Gc.abs())
        la = self.lin.abs()
        self.b_gv = self.b_gvc @ la + 4 * EPS * (self.g_vc.abs() @ la)
        kV = scatter_k(V) * EPS                 # the camera gradients sum over the vertices (library GEMM)
        ga = self.g_vc.abs()
        if mode == "T":
            top = va.transpose(1, 2) @ self.b_gvc + kV * (va.transpose(1, 2) @ ga)
            self.b_gcam = {"camera_transform": torch.cat([top, self.b_gvc.sum(1, keepdim=True) + kV * ga.sum(1, keepdim=True)], 1)}
        else:
            d = (va + ta)
            self.b_gcam = {"camera_rot": self.b_gvc.transpose(1, 2) @ d + kV * (ga.transpose(1, 2) @ d),
                           "camera_trans": ((self.b_gvc + kV * ga) @ la).sum(1).view_as(self.cam["camera_trans"])}


def run_pv(v, faces, mode, rot, trans, transform, w, proj=PROJ):
    tv = dev(v, True)
    cam = ({"camera_transform": dev(transform, True)} if mode == "T" else
           {"camera_rot": dev(rot, True), "camera_trans": dev(trans, True)})
    out = prepare_vertices(tv, faces.to(DEV), proj.to(DEV), **cam)
    if w is not None:
        sum((o * wi.to(DEV)).sum() for o, wi in zip(out, w) if wi is not None).backward()
    return out, tv, cam


def check_pv(v, faces, mode, rot, trans, transform, w, what, proj=PROJ):
    out, tv, cam = run_pv(v, faces, mode, rot, trans, transform, w, proj)
    ref = PV(v, faces, mode, rot, trans, transform, w, proj)
    for o, r, b, name in zip(out, ref.out, (ref.b_fvc, ref.b_fvi, ref.b_fn), ("fvc", "fvi", "fn")):
        within(o, r.detach(), b, f"{what} {mode} {name}")
    if w is not None:
        within(tv.grad, ref.g_v, ref.b_gv, f"{what} {mode} g_vertices")
        for k, t in cam.items():
            within(t.grad, ref.g_cam[k], ref.b_gcam[k], f"{what} {mode} g_{k}")
    return out, tv, cam, ref


def weights(B, F, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.rand((B, F, 3, 3), generator=g), torch.rand((B, F, 3, 2), generator=g), torch.rand((B, F, 3), generator=g)]


def gold_scene(tag):
    w = [torch.from_numpy(G[f"{tag}_w{i}"]) for i in (1, 2, 3)]
    return [torch.from_numpy(G[f"{tag}_{k}"]) for k in ("vertices", "faces")], \
        [torch.from_numpy(G[f"{tag}_{k}"]) for k in ("rot", "trans", "transform")], w


@pytest.mark.parametrize("mode", ["T", "Rt"])
def test_prepare_vertices_eps_scale(mode):
    """|e0 x e1| from 1e-13 to 1e-7: the 1e-10 in n = c / (L + 1e-10) and the L (L + 1e-10)^2 of its gradient
    decide the result.  Against float64 here and against the reference's own float64 numbers."""
    (v, faces), cam, w = gold_scene("ep")
    out, tv, tcam, ref = check_pv(v, faces, mode, *cam, w, "eps scale")
    assert ref.L.min() < 1e-13 and ref.L.max() > 1e-7 and ((ref.L > 1e-11) & (ref.L < 1e-9)).any()
    within(out[2], torch.from_numpy(G[f"ep_{mode}_fn"]), ref.b_fn, "eps scale fn vs reference")
    within(tv.grad, torch.from_numpy(G[f"ep_{mode}_g_vertices"]), ref.b_gv, "eps scale g_vertices vs reference")


@pytest.mark.parametrize("mode", ["T", "Rt"])
def test_prepare_vertices_degenerate_faces(mode):
    (v, faces), cam, w = gold_scene("dg")
    out, tv, tcam, ref = check_pv(v, faces, mode, *cam, w, "degenerate")
    deg = torch.from_numpy(G["dg_degenerate"])
    assert not out[2][:, deg.to(DEV)].any(), "normal of a zero-area face is exactly 0"
    assert torch.isfinite(tv.grad).all() and all(torch.isfinite(t.grad).all() for t in tcam.values())
    within(tv.grad, torch.from_numpy(G[f"dg_{mode}_g_vertices"]), ref.b_gv, "degenerate g_vertices vs reference")
    # the same mesh without them: the other faces' results do not change by a bit
    keep = torch.tensor([i for i in range(faces.shape[0]) if i not in set(deg.tolist())])
    out2, _, _ = run_pv(v, faces[keep], mode, *cam, None)
    for a, b in zip(out, out2):
        assert torch.equal(a[:, keep.to(DEV)], b)


@pytest.mark.parametrize("mode", ["T", "Rt"])
def test_prepare_vertices_fan_contention_and_unused_vertices(mode):
    """Vertex 0 is in every one of 120 000 faces, with two of 2000 others each (a fan in one ring would be all
    slivers); the last 5 vertices are in none."""
    g = torch.Generator().manual_seed(5)
    B, F, V = 2, 120_000, 1 + 2000 + 5
    v = torch.rand((B, V, 3), generator=g) - 0.5
    a = torch.randint(1, 2001, (F,), generator=g)
    faces = torch.stack([torch.zeros_like(a), a, 1 + (a - 1 + torch.randint(1, 2000, (F,), generator=g)) % 2000], 1)
    rot, trans = cameras(B, 6)
    out, tv, tcam, ref = check_pv(v, faces, mode, rot, trans, transform_of(rot, trans), weights(B, F, 7), "fan")
    assert not tv.grad[:, -5:].any(), "a vertex no face uses gets exactly 0"
    assert (tv.grad[:, 0].abs() > 100 * tv.grad[:, 1:-5].abs().mean()).all()       # the hub did collect


@pytest.mark.parametrize("mode", ["T", "Rt"])
def test_prepare_vertices_on_and_behind_the_camera_plane(mode):
    g = torch.Generator().manual_seed(8)
    B, V, F = 2, 60, 200
    v = torch.rand((B, V, 3), generator=g) - 0.5
    faces = torch.stack([torch.randperm(V, generator=g)[:3] for _ in range(F)])
    rot = torch.eye(3)[None].repeat(B, 1, 1)
    trans = torch.tensor([[0., 0., 2.], [0.25, 0., 2.]])
    clean = run_pv(v, faces, mode, rot, trans, transform_of(rot, trans), None)[0]
    v2 = v.clone()
    v2[:, 3] = torch.tensor([0.25, -0.5, 2.])        # on the camera plane: z = 0 exactly (0/0 in view 1's x)
    v2[:, 7] = torch.tensor([0., 0., 2.])            # the camera itself in view 0
    v2[:, 11] = torch.tensor([0.1, 0.2, 3.5])        # behind it
    out, tv, tcam, ref = check_pv(v2, faces, mode, rot, trans, transform_of(rot, trans), None, "camera plane")
    assert torch.isnan(out[1]).any() and torch.isinf(out[1]).any()
    untouched = ~torch.isin(faces, torch.tensor([3, 7, 11])).any(dim=1)
    assert 0 < untouched.sum() < F
    for a, b in zip(out, clean):
        assert torch.equal(a[:, untouched.to(DEV)], b[:, untouched.to(DEV)])


@pytest.mark.parametrize("B,F,V", [(1, 1, 3), (1, 255, 40), (2, 128, 40), (1, 257, 40), (3, 85, 1), (1, 7, 9)])
@pytest.mark.parametrize("mode", ["T", "Rt"])
def test_prepare_vertices_shapes(mode, B, F, V):
    """B*F either side of one 256-thread block, one vertex, one view."""
    g = torch.Generator().manual_seed(B * 1000 + F)
    v = torch.rand((B, V, 3), generator=g) - 0.5
    faces = torch.randint(0, V, (F, 3), generator=g)
    rot, trans = cameras(B, F)
    check_pv(v, faces, mode, rot, trans, transform_of(rot, trans), weights(B, F, 1), f"shape {B}x{F}x{V}")


@pytest.mark.parametrize("mode", ["T", "Rt"])
def test_prepare_vertices_empty_mesh(mode):
    B, V = 2, 5
    v = torch.rand((B, V, 3))
    rot, trans = cameras(B, 2)
    out, tv, tcam = run_pv(v, torch.zeros((0, 3), dtype=torch.int64), mode, rot, trans, transform_of(rot, trans), None)
    assert [tuple(o.shape) for o in out] == [(B, 0, 3, 3), (B, 0, 3, 2), (B, 0, 3)]
    (out[0].sum() + out[1].sum() + out[2].sum()).backward()
    assert tv.grad.shape == v.shape and not tv.grad.any() and all(not t.grad.any() for t in tcam.values())


def test_prepare_vertices_strided_inputs_and_translation_shapes():
    g = torch.Generator().manual_seed(12)
    B, V, F = 3, 30, 50
    v = torch.rand((B, V, 3), generator=g) - 0.5
    faces = torch.randint(0, V, (F, 3), generator=g)
    rot, trans = cameras(B, 3)
    T = transform_of(rot, trans)
    w = [x.to(DEV) for x in weights(B, F, 2)]
    loss = lambda o: sum((a * b).sum() for a, b in zip(o, w))
    base = {}
    for mode, kw in (("T", dict(camera_transform=dev(T, True))), ("Rt", dict(camera_rot=dev(rot, True), camera_trans=dev(trans, True)))):
        tv = dev(v, True)
        o = prepare_vertices(tv, faces.to(DEV), PROJ.to(DEV), **kw)
        loss(o).backward()
        base[mode] = (o, tv.grad, {k: t.grad for k, t in kw.items()})
    # the same values behind strides: vertices as a slice of a wider buffer, cameras transposed in memory
    wide = torch.zeros((B, V, 6), device=DEV); wide[..., ::2] = dev(v)
    sv = wide[..., ::2].requires_grad_(True)
    sT = dev(T).transpose(1, 2).contiguous().transpose(1, 2).requires_grad_(True)
    sR = dev(rot).transpose(1, 2).contiguous().transpose(1, 2).requires_grad_(True)
    sf = torch.stack([faces.to(DEV), faces.to(DEV)], -1)[..., 0]
    assert not sv.is_contiguous() and not sT.is_contiguous() and not sR.is_contiguous() and not sf.is_contiguous()
    for mode, kw in (("T", dict(camera_transform=sT)), ("Rt", dict(camera_rot=sR, camera_trans=dev(trans.view(B, 1, 3), True)))):
        sv.grad = None
        o = prepare_vertices(sv, sf, PROJ.to(DEV), **kw)
        loss(o).backward()
        bo = base[mode][0]
        assert all(torch.equal(a, b) for a, b in zip(o, bo))
        # gradients against float64 rather than against the contiguous run: the scatter's atomics add a vertex's
        # corners in any order, and those corners cancel
        ref = PV(v, faces, mode, rot, trans, T, [x.cpu() for x in w])
        within(sv.grad, ref.g_v, ref.b_gv, f"strided {mode} g_vertices")
        within(base[mode][1], ref.g_v, ref.b_gv, f"contiguous {mode} g_vertices")
        for k, t in kw.items():
            assert t.grad.shape == t.shape
            within(t.grad.reshape(ref.g_cam[k].shape), ref.g_cam[k], ref.b_gcam[k], f"strided {mode} g_{k}")


@pytest.mark.parametrize("mode", ["T", "Rt"])
def test_prepare_vertices_gradient_subsets(mode):
    """Each non-empty subset of the three output gradients, the rest NULL (entry point) or unused
    (autograd): equal to the full call with zeros in those slots, and to float64."""
    g = torch.Generator().manual_seed(21)
    B, V, F = 2, 200, 300         # ~4.5 corners per vertex
    v = torch.rand((B, V, 3), generator=g) - 0.5
    faces = torch.stack([torch.randperm(V, generator=g)[:3] for _ in range(F)])
    rot, trans = cameras(B, 4)
    T = transform_of(rot, trans)
    w = weights(B, F, 3)
    tv, tf = dev(v), faces.to(DEV)
    cam = (dev(T), None, None) if mode == "T" else (None, dev(rot), dev(trans))
    proj = (__import__("ctypes").c_float * 3)(*PROJ.reshape(-1).tolist())
    gs = [x.to(DEV) for x in w]

    def entry(grads):
        out = torch.empty((B, V, 3), device=DEV)
        _lib.call("dibr_b200_prepare_vertices_backward", tv.device, B, V, F, tv, tf, *cam, proj, *grads, out)
        return out

    for mask in range(1, 8):
        on = [bool(mask >> i & 1) for i in range(3)]
        null = entry([x if o else None for x, o in zip(gs, on)])
        zero = entry([x if o else torch.zeros_like(x) for x, o in zip(gs, on)])
        sub = [x if o else None for x, o in zip(w, on)]
        ref = PV(v, faces, mode, rot, trans, T, sub)
        within(null, ref.g_vc, ref.b_gvc, f"subset {on} {mode} NULL slots vs float64")
        within(zero, ref.g_vc, ref.b_gvc, f"subset {on} {mode} zeros in the slots vs float64")
        _, av, acam = run_pv(v, faces, mode, rot, trans, T, sub)          # through autograd: unused outputs
        within(av.grad, ref.g_v, ref.b_gv, f"subset {on} {mode} autograd g_vertices")
        for k, t in acam.items():
            within(t.grad, ref.g_cam[k], ref.b_gcam[k], f"subset {on} {mode} autograd g_{k}")


def test_prepare_vertices_rejects_non_float32():
    v = torch.rand((1, 4, 3), device=DEV)
    f = torch.tensor([[0, 1, 2]], device=DEV)
    rot, trans = cameras(1, 1)
    T = transform_of(rot, trans).to(DEV)
    for bad in (v.to(torch.int32), v > 0.5, v.long(), v.double(), v.half()):
        with pytest.raises(RuntimeError, match="not implemented for"):
            prepare_vertices(bad, f, PROJ.to(DEV), camera_transform=T)
    with pytest.raises(RuntimeError, match="not implemented for"):
        prepare_vertices(v, f, PROJ.to(DEV), camera_transform=T.to(torch.int64))
    with pytest.raises(RuntimeError, match="not implemented for"):
        prepare_vertices(v, f, PROJ.to(DEV), camera_rot=rot.to(DEV), camera_trans=trans.to(DEV).to(torch.int32))
    with pytest.raises(NotImplementedError):
        prepare_vertices(v, f.to(torch.int32), PROJ.to(DEV), camera_transform=T)


# =================================================================================================
# texture_mapping
def source_index(c32, size, flip):
    """Where float32 coordinates land on an axis of `size` texels: the float64 source index after the
    border clip, and whether float32 arithmetic is sure to land in the same half-texel: either its
    chain (clamp, 2u - 1, flip, one fused (g + 1) size - 1, halve) is exact on this input, or the index
    is further from every multiple of 0.5 than that chain's error, 3 EPS size (2u - 1 rounds by EPS at
    most, which size / 2 magnifies; the fused step rounds by EPS size at most)."""
    c32 = c32.detach().cpu().float()
    c = c32.double().clamp(0, 1)
    g = c * 2 - 1
    i = (((-g if flip else g) + 1) * size - 1) / 2
    g3 = c32.clamp(0, 1) * 2 - 1
    s3 = (-g3 if flip else g3) + 1
    i3 = (s3.double() * size - 1).float() * 0.5
    ic, i3c = i.clamp(0, size - 1), i3.double().clamp(0, size - 1)
    far = ((ic * 2) - (ic * 2).round()).abs() / 2 > 3 * EPS * size
    return ic, (i3c == ic) | far


class TM:
    """float64 texture_mapping of float32 inputs with per-element bounds.  `sure`: the points where float32
    and float64 select the same texels (see source_index); elsewhere only the library in float32 judges."""

    def __init__(self, uv, tex, gw, mode, nmax=None):
        self.mode = mode
        u, t = f64(uv).requires_grad_(True), f64(tex).requires_grad_(True)
        B, C, Ht, Wt = t.shape
        self.out = P.texture_mapping_torch(u, t, mode=mode)
        (self.out * f64(gw)).sum().backward()
        self.out = self.out.detach()
        self.g_tex = t.grad
        self.g_uv = u.grad if u.grad is not None else torch.zeros_like(u)
        flat = uv.detach().cpu().reshape(B, -1, 2)
        N = flat.shape[1]
        _, su = source_index(flat[..., 0], Wt, False)
        _, sv = source_index(flat[..., 1], Ht, True)
        self.sure = (su & sv).reshape(uv.shape[:-1])
        ta = t.detach().abs().amax(dim=(2, 3))                       # (B,C)
        rng = t.detach().amax(dim=(2, 3)) - t.detach().amin(dim=(2, 3))
        ga = f64(gw).abs().reshape(B, N, C)
        dix, diy = 3 * EPS * Wt, 3 * EPS * Ht                        # float32 error of the source index
        if mode == "nearest":
            self.b_out = torch.zeros(())                              # a copy of one texel
        else:
            # four products and three sums of |.| <= max|tex| (8 EPS), and weights off by the index error
            # times the largest step between neighbouring texels (<= the texture's range)
            self.b_out = ((dix + diy) * rng + 8 * EPS * ta)[:, None, :].expand(B, N, C).reshape(self.out.shape)
        # g_tex: each texel sums g * weight over the samples that touch it.  A = that sum with |g| (the weights
        # are >= 0), from the float64 side; accumulated by atomics (scatter_k of the samples per texel, at most
        # nmax); a weight is off by the index error, which moves |g| (dix + diy) between the corners of a sample,
        # all of them within the 3x3 block around any one of them
        u2 = f64(uv)
        t2 = torch.zeros_like(t).requires_grad_(True)
        (P.texture_mapping_torch(u2, t2, mode=mode) * f64(gw).abs()).sum().backward()
        A = t2.grad
        box = torch.nn.functional.avg_pool2d(A, 3, stride=1, padding=1, divisor_override=1) if mode == "bilinear" else 0 * A
        self.b_gtex = scatter_k(N if nmax is None else nmax) * EPS * A + (dix + diy) * box
        # g_uv = size * sum_c g_c * (difference of two texel pairs blended by the other axis' weights):
        # ~6 roundings per channel on |g| * 2 max|tex|, and the blend weight off by the other axis' index error
        gsum = (ga * (16 * EPS * ta + 2 * max(dix, diy) * rng)[:, None, :]).sum(-1)
        self.b_guv = torch.stack([gsum * Wt, gsum * Ht], -1).reshape(self.g_uv.shape)


def run_tm(uv, tex, gw, mode, grad_uv=True, grad_tex=True):
    tu, tt = dev(uv, grad_uv), dev(tex, grad_tex)
    o = texture_mapping(tu, tt, mode=mode)
    if grad_uv or grad_tex:
        (o * gw.to(DEV)).sum().backward()
    return o, tu.grad, tt.grad


def check_tm(uv, tex, gw, mode, what, nmax=None):
    o, g_uv, g_tex = run_tm(uv, tex, gw, mode)
    ref = TM(uv, tex, gw, mode, nmax)
    sure = ref.sure
    assert sure.float().mean() > 0.5, what
    # outputs and coordinate gradients where both precisions select the same texels
    m = sure[..., None].expand_as(ref.out)
    within(torch.where(m.to(DEV), o, torch.zeros_like(o)), torch.where(m, ref.out, torch.zeros_like(ref.out)), ref.b_out, f"{what} {mode} out")
    m = sure[..., None].expand_as(ref.g_uv)
    within(torch.where(m.to(DEV), g_uv, torch.zeros_like(g_uv)), torch.where(m, ref.g_uv, torch.zeros_like(ref.g_uv)), ref.b_guv, f"{what} {mode} g_uv")
    assert torch.equal((f64(g_uv) == 0) | ~m, (ref.g_uv == 0) | ~m), f"{what} {mode}: g_uv exactly 0 in the clamp and border zones"
    if bool(sure.all()):
        within(g_tex, ref.g_tex, ref.b_gtex, f"{what} {mode} g_tex")
        assert not g_tex[(ref.b_gtex == 0).to(DEV)].any(), f"{what} {mode}: a texel no sample touches gets exactly 0"
    return (o, g_uv, g_tex), ref


def vs_library(uv, tex, gw, mode, what):
    """Against torch's CUDA grid_sample in float32: the same texels, so outputs and gradients to the last bits."""
    o, g_uv, g_tex = run_tm(uv, tex, gw, mode)
    ru, rt = dev(uv, True), dev(tex, True)
    ro = P.texture_mapping_torch(ru, rt, mode=mode)
    (ro * gw.to(DEV)).sum().backward()
    r_guv = ru.grad if ru.grad is not None else torch.zeros_like(ru)
    if mode == "nearest":
        assert torch.equal(o, ro), f"{what}: nearest texel differs from grid_sample on {int((o != ro).any(-1).sum())} points"
    else:
        # the same source index gives the same weights; the two kernels order their four-term sums differently
        within(o, f64(ro), 8 * EPS * f64(tex).abs().max(), f"{what} bilinear out vs grid_sample")
    assert torch.equal(g_uv == 0, r_guv == 0), f"{what} {mode}: zero pattern of g_uv differs from grid_sample"
    size = max(tex.shape[-2:])
    within(g_uv, f64(r_guv), 32 * EPS * size * f64(gw).abs().sum(-1).max() * f64(tex).abs().max(), f"{what} {mode} g_uv vs grid_sample")
    return o, ro


def lattice(size):
    """Every texel boundary j / size (0 and 1 included) and every texel centre (j + 0.5) / size."""
    return torch.cat([torch.arange(size + 1, dtype=D) / size, (torch.arange(size, dtype=D) + 0.5) / size]).float()


def pairs(us, vs):
    return torch.stack(torch.meshgrid(us, vs, indexing="ij"), -1).reshape(1, -1, 2)


def index_texture(Ht, Wt):
    """Channel 0 holds each texel's column, channel 1 its row: 'nearest' returns the texel it picked and
    'bilinear' the source index it computed."""
    y, x = torch.meshgrid(torch.arange(Ht, dtype=torch.float32), torch.arange(Wt, dtype=torch.float32), indexing="ij")
    return torch.stack([x, y])[None]


@pytest.mark.parametrize("Ht,Wt", [(4, 8), (64, 32)])
def test_texture_mapping_lattice_exact(Ht, Wt):
    """Power-of-two sizes: the source index of every boundary and centre is exact in float32 (j - 0.5 and j),
    so the result is known exactly: nearest rounds the ties half to even, bilinear returns a centre's texel
    bit for bit and the correctly rounded mean on a boundary between two centres."""
    g = torch.Generator().manual_seed(Ht)
    uv = pairs(lattice(Wt), lattice(Ht))
    ix = (uv[..., 0].double() * Wt - 0.5).clamp(0, Wt - 1)
    iy = ((1 - uv[..., 1].double()) * Ht - 0.5).clamp(0, Ht - 1)
    o = texture_mapping(uv.to(DEV), index_texture(Ht, Wt).to(DEV), mode="nearest").cpu()
    assert torch.equal(o[..., 0].double(), torch.from_numpy(np.rint(ix.numpy()))), "column: half to even"
    assert torch.equal(o[..., 1].double(), torch.from_numpy(np.rint(iy.numpy()))), "row: half to even"
    assert (np.rint(ix.numpy()) != np.floor(ix.numpy() + 0.5)).any()       # ties that round() would send the other way
    tex = torch.rand((1, 3, Ht, Wt), generator=g)
    o = texture_mapping(uv.to(DEV), tex.to(DEV), mode="bilinear").cpu()
    x0, y0 = ix.floor().long(), iy.floor().long()
    x1, y1 = (x0 + 1).clamp(max=Wt - 1), (y0 + 1).clamp(max=Ht - 1)
    fx, fy = (ix - x0)[..., None], (iy - y0)[..., None]
    t = tex[0].double().permute(1, 2, 0)
    mean = (t[y0, x0] * (1 - fx) + t[y0, x1] * fx) * (1 - fy) + (t[y1, x0] * (1 - fx) + t[y1, x1] * fx) * fy
    one_axis = ((fx == 0) | (fy == 0)).expand_as(mean)      # a centre along at least one axis: at most one rounding
    assert (fx == 0).any() and (fx == 0.5).any() and (fy == 0.5).any()
    assert torch.equal(o[one_axis], mean.float()[one_axis]), "centres bit for bit, boundaries the rounded mean"
    within(o, mean, 4 * EPS * mean.abs(), "corner of four texels")
    for mode in MODES:
        gw = torch.rand((1, uv.shape[1], 3), generator=g)
        (_, g_uv, _), ref = check_tm(uv, tex, gw, mode, f"lattice {Ht}x{Wt}")
        assert bool(ref.sure.all())


@pytest.mark.parametrize("Ht,Wt", [(7, 9), (96, 100), (1000, 3), (3, 1000)])
@pytest.mark.parametrize("mode", MODES)
def test_texture_mapping_lattice_vs_library(mode, Ht, Wt):
    """Sizes that are not powers of two: the source index is rounded, and which way depends on how
    (g + 1) * size - 1 is evaluated.  The texel picked on every boundary and centre, and the source index
    itself (the bilinear sample of the index texture), equal those of torch's CUDA grid_sample."""
    g = torch.Generator().manual_seed(Wt)
    us, vs = lattice(Wt), lattice(Ht)
    if us.numel() * vs.numel() > 200_000:
        us = us[::3]
    uv = pairs(us, vs)
    gw = torch.rand((1, uv.shape[1], 2), generator=g)
    o, ro = vs_library(uv, index_texture(Ht, Wt), gw, mode, f"lattice {Ht}x{Wt}")
    if mode == "bilinear":      # the blend of a row / column index with its neighbour IS the source index,
        # up to the roundings of the two kernels' four-term sums (each within an ulp, 2 EPS relative)
        within(o, f64(ro), 8 * EPS * f64(ro).abs() + 1e-30, f"lattice {Ht}x{Wt} source index vs grid_sample")


def kinks(size):
    h, one = np.float32(0.5 / size), np.float32(1)
    up = lambda x: np.nextafter(np.float32(x), np.float32(np.inf))
    dn = lambda x: np.nextafter(np.float32(x), np.float32(-np.inf))
    d = np.float32(2.0 ** -24)        # the step of 2u - 1 near +-1: what the grid coordinate resolves
    return torch.from_numpy(np.array(
        [-1., -0., 0., 1e-40, dn(h), h, up(h), h - d, h + d, dn(one - h), one - h, up(one - h), one - h - d, one - h + d,
         0.5, 0.3, one - d, 1., 1. + 2.0 ** -23, 2., np.inf, -np.inf], np.float32))


@pytest.mark.parametrize("tag", ["tk51", "tk48"])
@pytest.mark.parametrize("mode", MODES)
def test_texture_mapping_kinks_vs_reference_float64(mode, tag):
    """Every pair of kink coordinates, against the reference's own float64 numbers where float32 resolves
    the coordinate (on the 4x8 texture all but the +-1 ulp neighbours of half a texel), against
    grid_sample in float32 everywhere."""
    uv, tex, gw = (torch.from_numpy(G[f"{tag}_{k}"]) for k in ("uv", "tex", "gw"))
    (o, g_uv, g_tex), ref = check_tm(uv, tex, gw, mode, f"kinks {tag}")
    for k, a in (("out", ref.out), ("g_uv", ref.g_uv), ("g_tex", ref.g_tex)):
        assert (a - torch.from_numpy(G[f"{tag}_{mode}_{k}"])).abs().max() <= 1e-12
    if mode == "bilinear":
        assert (f64(g_uv)[ref.sure] != 0).any() and (f64(g_uv)[ref.sure] == 0).any()
    vs_library(uv, tex, gw, mode, f"kinks {tag}")


@pytest.mark.parametrize("Ht,Wt", [(1, 1), (1, 5), (5, 1), (2, 2), (3, 6)])
@pytest.mark.parametrize("mode", MODES)
def test_texture_mapping_kinks_small_textures(mode, Ht, Wt):
    """A texture one texel wide has no right-hand neighbour anywhere: every x1 / y1 corner is dropped."""
    g = torch.Generator().manual_seed(Ht * 10 + Wt)
    uv = pairs(kinks(Wt), kinks(Ht)).repeat(3, 1, 1)
    tex = torch.rand((3, 2, Ht, Wt), generator=g) * 2 - 1             # differs per batch entry
    gw = torch.rand((3, uv.shape[1], 2), generator=g) - 0.3
    check_tm(uv, tex, gw, mode, f"kinks {Ht}x{Wt}")
    vs_library(uv, tex, gw, mode, f"kinks {Ht}x{Wt}")


@pytest.mark.parametrize("mode", MODES)
def test_texture_mapping_nan_coordinate_reads_as_zero(mode):
    """Pinned, deliberate difference from grid_sample: NaN is read as coordinate 0 and gets no gradient."""
    g = torch.Generator().manual_seed(4)
    tex = torch.rand((1, 3, 5, 6), generator=g)
    nan = float("nan")
    uv = torch.tensor([[[nan, 0.3], [0.7, nan], [nan, nan], [0.7, 0.3]]])
    as0 = torch.tensor([[[0., 0.3], [0.7, 0.], [0., 0.], [0.7, 0.3]]])
    gw = torch.rand((1, 4, 3), generator=g)
    o, g_uv, g_tex = run_tm(uv, tex, gw, mode)
    o0, g_uv0, g_tex0 = run_tm(as0, tex, gw, mode)
    assert torch.equal(o, o0) and torch.equal(g_tex, g_tex0)
    assert torch.equal(o[0, 2], tex[0, :, 4, 0].to(DEV)), "u = 0: leftmost column, v = 0: bottom row"
    assert not g_uv[0, 0, 0].item() and not g_uv[0, 1, 1].item() and not g_uv[0, 2].any()
    assert torch.equal(g_uv[0, 3], g_uv0[0, 3]) and torch.equal(g_uv[0, 0, 1], g_uv0[0, 0, 1])


@pytest.mark.parametrize("C", [1, 2, 3, 4, 7, 64])
@pytest.mark.parametrize("mode", MODES)
def test_texture_mapping_channels_and_batches(mode, C):
    g = torch.Generator().manual_seed(C)
    B, N, Ht, Wt = 3, 301, 6, 10
    uv = torch.rand((B, N, 2), generator=g) * 1.2 - 0.1
    tex = torch.rand((B, C, Ht, Wt), generator=g) * 2 - 1
    check_tm(uv, tex, torch.rand((B, N, C), generator=g) - 0.5, mode, f"C={C}")


@pytest.mark.parametrize("shape", [(0,), (1,), (255,), (256,), (257,), (7, 9), (1, 1), (17, 15)])
@pytest.mark.parametrize("mode", MODES)
def test_texture_mapping_point_counts_and_dense_shapes(mode, shape):
    g = torch.Generator().manual_seed(len(shape) * 100 + shape[0])
    B, C = 2, 3
    uv = torch.rand((B, *shape, 2), generator=g) * 1.2 - 0.1
    tex = torch.rand((B, C, 4, 8), generator=g)
    gw = torch.rand((B, *shape, C), generator=g)
    if shape == (0,):
        o, g_uv, g_tex = run_tm(uv, tex, gw, mode)
        assert o.shape == (B, 0, C) and g_uv.shape == uv.shape and not g_tex.any()
        return
    (o, _, _), _ = check_tm(uv, tex, gw, mode, f"points {shape}")
    assert o.shape == (B, *shape, C)


@pytest.mark.parametrize("mode", MODES)
def test_texture_mapping_hot_texel(mode):
    """2^20 samples inside the footprint of one texel of a 16x16 texture."""
    g = torch.Generator().manual_seed(33)
    N, S, C = 1 << 20, 16, 2
    # centre of texel (row 5 from the top, column 9), +-0.45 texel: bilinear touches the 3x3 block around it
    uv = torch.stack([(9.5 + 0.9 * (torch.rand(N, generator=g) - 0.5)) / S,
                      1 - (5.5 + 0.9 * (torch.rand(N, generator=g) - 0.5)) / S], -1)[None]
    tex = torch.rand((1, C, S, S), generator=g)
    gw = torch.rand((1, N, C), generator=g)
    (o, g_uv, g_tex), ref = check_tm(uv, tex, gw, mode, "hot texel", nmax=N)
    foot = torch.zeros((S, S), dtype=torch.bool)
    if mode == "nearest":
        foot[5, 9] = True
        assert not g_uv.any()
        hist = f64(gw).sum(1)[0]                     # every sample lands on the one texel: a float64 histogram
        within(g_tex[0, :, 5, 9], hist, scatter_k(N) * EPS * hist, "hot texel histogram")
    else:
        foot[4:7, 8:11] = True
    assert not g_tex[:, :, ~foot.to(DEV)].any(), "texels outside the footprint get exactly 0"
    assert (g_tex[:, :, foot.to(DEV)] != 0).all()


@pytest.mark.parametrize("grad_uv,grad_tex", [(True, False), (False, True), (False, False)])
@pytest.mark.parametrize("mode", MODES)
def test_texture_mapping_requires_grad_combinations(mode, grad_uv, grad_tex):
    g = torch.Generator().manual_seed(44)
    uv = torch.rand((2, 100, 2), generator=g) * 1.2 - 0.1
    tex = torch.rand((2, 3, 5, 7), generator=g)
    gw = torch.rand((2, 100, 3), generator=g)
    full = run_tm(uv, tex, gw, mode)
    o, g_uv, g_tex = run_tm(uv, tex, gw, mode, grad_uv, grad_tex)
    assert torch.equal(o, full[0]) and o.requires_grad == (grad_uv or grad_tex)
    assert (g_uv is not None) == grad_uv and (g_tex is not None) == grad_tex
    if grad_uv:
        assert torch.equal(g_uv, full[1])
    if grad_tex:
        within(g_tex, f64(full[2]), scatter_k(100) * EPS * f64(full[2]).abs() + 1e-30, "g_tex alone")


@pytest.mark.parametrize("mode", MODES)
def test_texture_mapping_misaligned_coordinates(mode):
    """A contiguous view 4 bytes past an 8-byte boundary (legal input, not copied by .contiguous()):
    the same bits as its aligned clone.  One point per texel at most, so no atomic order to differ."""
    g = torch.Generator(device=DEV); g.manual_seed(9)
    B, N, S = 2, 37, 32
    buf = torch.rand(B * N * 2 + 3, device=DEV, generator=g)
    uv = buf[1:1 + 2 * B * N].view(B, N, 2)
    assert uv.data_ptr() % 8 == 4 and uv.is_contiguous()
    tex = torch.rand((B, 3, S, S), device=DEV, generator=g)
    gw = torch.rand((B, N, 3), device=DEV, generator=g)
    res = []
    for c in (uv, uv.clone()):
        c = c.detach().requires_grad_(True)
        t = tex.clone().requires_grad_(True)
        o = texture_mapping(c, t, mode=mode)
        (o * gw).sum().backward()
        res.append((o, c.grad, t.grad))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    within(res[0][2], f64(res[1][2]), 8 * EPS * f64(res[1][2]).abs() + 1e-30, "misaligned g_tex")
    ref = P.texture_mapping_torch(f64(uv), f64(tex), mode=mode)
    within(res[0][0], ref, 16 * EPS * S, "misaligned out vs float64")


def test_texture_mapping_rejects_non_float32():
    uv = torch.rand((1, 5, 2), device=DEV)
    tex = torch.rand((1, 3, 4, 4), device=DEV)
    for bad in (uv.long(), uv > 0.5, uv.to(torch.uint8), uv.double(), uv.bfloat16()):
        with pytest.raises(RuntimeError, match="not implemented for"):
            texture_mapping(bad, tex)
    for bad in ((tex * 255).to(torch.uint8), tex.long(), tex.half()):
        with pytest.raises(RuntimeError, match="not implemented for"):
            texture_mapping(uv, bad)


# =================================================================================================
# mask_iou
def check_iou(l, r, what, grad_l=True, grad_r=True, upstream=1.0, loss_tol=None):
    """Loss and gradients against float64.  The kernel's per-view sums run over HW terms: 8 per thread in
    sequence, a tree over the block, one atomic per block (scatter_k of the blocks): (16 + scatter_k) EPS
    times the sum of |terms|, where a term of the union, (l + r) - l r, is itself rounded twice."""
    tl, tr = dev(l, grad_l), dev(r, grad_r)
    loss = mask_iou(tl, tr)
    assert loss.shape == () and loss.dtype == torch.float32
    l64, r64 = f64(l).requires_grad_(True), f64(r).requires_grad_(True)
    ref = P.mask_iou_torch(l64, r64)
    B, HW = l.shape[0], l[0].numel()
    blocks = min((HW + 2047) // 2048, 1056)
    rel = (16 + scatter_k(blocks)) * EPS
    a, c = l64.detach().reshape(B, -1), r64.detach().reshape(B, -1)
    up, de = (a * c).sum(1), (a + c - a * c).sum(1) + 1e-10
    b_up = rel * (a * c).abs().sum(1)
    b_de = rel * (a.abs() + c.abs() + (a * c).abs()).sum(1) + 2 * EPS * 1e-10
    b_iou = b_up / de.abs() + up.abs() * b_de / de ** 2 + 2 * EPS * (up / de).abs()
    b_loss = b_iou.mean() + 4 * EPS
    within(loss, ref.detach(), b_loss if loss_tol is None else min(float(b_loss), loss_tol), f"{what} loss")
    if not (grad_l or grad_r):
        assert not loss.requires_grad
        return loss
    (loss * upstream).backward()
    (ref * upstream).backward()
    k = (upstream / (B * de ** 2)).abs()[:, None]
    for on, t, g64, own, other in ((grad_l, tl, l64.grad, a, c), (grad_r, tr, r64.grad, c, a)):
        if not on:
            assert t.grad is None
            continue
        # g = -k (other de - up (1 - other)), k = upstream / (B de^2): the sums' errors carried through, and ~6
        # roundings on the two terms
        terms = other.abs() * de.abs()[:, None] + up.abs()[:, None] * (1 - other).abs()
        bound = k * (other.abs() * b_de[:, None] + (1 - other).abs() * b_up[:, None] + 8 * EPS * terms) \
            + 2 * g64.reshape(B, -1).abs() * (b_de / de.abs())[:, None]
        within(t.grad.reshape(B, -1), g64.reshape(B, -1), bound, f"{what} g_{'lhs' if t is tl else 'rhs'}")
    return loss


def masks(shape, seed, soft=True):
    g = torch.Generator().manual_seed(seed)
    l = torch.rand(shape, generator=g)
    r = (torch.rand(shape, generator=g) > 0.6).float()
    return (l if soft else (l > 0.5).float()), r


@pytest.mark.parametrize("shape", [(3, 1, 1), (2, 1, 255), (2, 257, 1), (3, 23, 89), (2, 2049, 1), (65535, 2, 2),
                                   (1, 1536, 1536)])
def test_mask_iou_shapes(shape):
    """One pixel, either side of a 256-thread block and of its 2048 pixels, the largest batch the grid
    takes, and a view above 1056 * 2048 pixels, where each thread strides more than once."""
    l, r = masks(shape, shape[1])
    check_iou(l, r, f"shape {shape}", upstream=0.7)


def test_mask_iou_benchmark_size():
    l, r = masks((32, 1024, 1024), 1)
    check_iou(l, r, "32x1024x1024", loss_tol=1e-6)


def test_mask_iou_too_many_views():
    l = torch.zeros((65536, 1, 2), device=DEV)
    with pytest.raises(RuntimeError, match="65535"):
        mask_iou(l, l)


def test_mask_iou_strided_masks():
    l, r = masks((3, 20, 34), 5)
    tl, tr = dev(l, True), dev(r)
    sl, sr = tl[..., ::2], tr[:, ::2]
    assert not sl.is_contiguous() and not sr.is_contiguous()
    a = mask_iou(sl, tr[..., ::2])
    a.backward()
    cl = dev(l[..., ::2], True)
    b = mask_iou(cl, dev(r[..., ::2]))
    b.backward()
    assert tl.grad.shape == l.shape and not tl.grad[..., 1::2].any()
    within(a, f64(b), 4 * EPS, "strided loss")
    within(tl.grad[..., ::2], f64(cl.grad), 16 * EPS * f64(cl.grad).abs() + 1e-30, "strided g_lhs")
    check_iou(l[..., ::2], r[..., ::2], "strided values")


@pytest.mark.parametrize("name", ["empty", "full", "one_empty", "complement", "range"])
def test_mask_iou_values_vs_reference_float64(name):
    l, r = torch.from_numpy(G[f"mi_{name}_lhs"]), torch.from_numpy(G[f"mi_{name}_rhs"])
    scale = float(G["mi_gscale"])
    tl, tr = dev(l, True), dev(r, True)
    loss = mask_iou(tl, tr)
    (loss * scale).backward()
    check_iou(l, r, name, upstream=scale)
    if name != "range":       # there the sums cancel, and only check_iou's bound (sum of |terms|) applies
        assert abs(loss.item() - float(G[f"mi_{name}_loss"])) <= 1e-6
    for t, k in ((tl, "lhs"), (tr, "rhs")):
        ref = torch.from_numpy(G[f"mi_{name}_g_{k}"])
        within(t.grad, ref, 1e-5 * ref.abs() + 1e-6 * ref.abs().max(), f"{name} g_{k} vs reference")
    if name == "empty":
        assert loss.item() == 1.0 and not tl.grad.any() and not tr.grad.any()
    if name == "complement":
        assert loss.item() == 1.0


def test_mask_iou_large_values():
    """Nothing clamps: masks in [-2, 2) and [-1, 2) over a real image size."""
    g = torch.Generator().manual_seed(17)
    check_iou(torch.rand((2, 200, 300), generator=g) * 4 - 2, torch.rand((2, 200, 300), generator=g) * 3 - 1, "range")


@pytest.mark.parametrize("grad_l,grad_r", [(True, False), (False, True), (True, True), (False, False)])
def test_mask_iou_gradient_subsets(grad_l, grad_r):
    l, r = masks((3, 40, 50), 8)
    r = 0.2 + 0.6 * r
    check_iou(l, r, f"grads {grad_l},{grad_r}", grad_l, grad_r, upstream=-2.5)


def test_mask_iou_loss_used_twice():
    l, r = masks((2, 30, 30), 9)
    tl = dev(l, True)
    loss = mask_iou(tl, dev(r))
    (loss * loss + 3 * loss).backward()
    l64 = f64(l).requires_grad_(True)
    ref = P.mask_iou_torch(l64, f64(r))
    (ref * ref + 3 * ref).backward()
    within(tl.grad, l64.grad, 1e-5 * l64.grad.abs() + 64 * EPS * l64.grad.abs().max(), "loss used twice")


@pytest.mark.parametrize("dtype", [torch.bool, torch.uint8, torch.int32, torch.int64])
@pytest.mark.parametrize("side", ["rhs", "lhs", "both"])
def test_mask_iou_integer_and_bool_masks(side, dtype):
    """Converted to float32, as the reference promotes them; the converted mask gets no gradient."""
    l, r = masks((3, 33, 47), 3, soft=False)
    if dtype not in (torch.bool,):
        r, l = r * 2, l * 3 if side != "rhs" else l         # integer masks need not be 0 / 1
    soft = torch.rand(l.shape, generator=torch.Generator().manual_seed(4))
    fl, fr = (l if side in ("lhs", "both") else soft), (r if side in ("rhs", "both") else soft)
    tl = fl.to(DEV, dtype) if side in ("lhs", "both") else dev(fl, True)
    tr = fr.to(DEV, dtype) if side in ("rhs", "both") else dev(fr, True)
    loss = mask_iou(tl, tr)
    cl, cr = dev(fl, side == "rhs"), dev(fr, side == "lhs")
    ref = mask_iou(cl, cr)
    assert torch.equal(loss, ref) or abs(loss.item() - ref.item()) <= 4 * EPS     # per-view sums are atomics
    check_iou(fl, fr, f"{dtype} {side}", grad_l=False, grad_r=False)
    if side == "both":
        assert not loss.requires_grad
        return
    loss.backward(); ref.backward()
    t, c = (tl, cl) if side == "rhs" else (tr, cr)
    within(t.grad, f64(c.grad), 16 * EPS * f64(c.grad).abs() + 1e-30, f"{dtype} {side} gradient of the float mask")


def test_mask_iou_rejects_other_floating_types():
    l = torch.rand((2, 4, 4), device=DEV)
    for bad in (l.double(), l.half(), l.bfloat16()):
        with pytest.raises(RuntimeError, match="not implemented for"):
            mask_iou(bad, l)
        with pytest.raises(RuntimeError, match="not implemented for"):
            mask_iou(l, bad)
