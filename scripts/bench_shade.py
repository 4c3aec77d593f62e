"""Deferred shading (sg_shade, kaolin_b200/csrc/lighting.cu kind SHADE) against two torch paths on one
GPU: a G-buffer of B views at H x W, L lights.

    python scripts/bench_shade.py [--views 8] [--res 1024] [--lights 1,8,32,128] [--min-seconds 0.5]

The G-buffer: per view a disc-shaped silhouette (about half of the pixels covered, the rest background,
as an object in the middle of the frame gives), normals with n.v in [0.25, 1] of each pixel's view,
albedo and spec_albedo from the metallic-roughness workflow, roughness in [0.3, 1].  For every L:
CUDA-event times of the forward, of forward+backward with all gradients and of forward+backward with
light gradients only, for
  * "ours":     the fused sg_shade;
  * "composed": the reference's sg_shade structure on this library's sg_diffuse_inner_product and
                sg_warp_specular_term, with boolean gathers and scatters;
  * "torch":    the reference formulation in fp32 torch (oracle/shade.py).
Both torch paths are given the per-pixel view grid, computed once before timing: their times leave
out the reference's per-call ray generation, so they are lower bounds for its structure.
The output and every gradient are checked against the fp64 restatement over every covered pixel of the
first view, next to the fp32 formulation's error; the script fails where an error exceeds both 1e-5 of
scale and 4x the fp32 formulation's.  It reports a byte model (face_idx read for every pixel; normal,
albedo, spec albedo and roughness read for covered pixels; three images written), the binding limit
(HBM bytes at 3.35 TB/s, or SFU issue at the SM clock), the fraction of it reached, the coverage, the
device name and power limit, then one JSON line.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time
import types

import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
from oracle import shade as OSH  # noqa: E402
from kaolin_b200.render import easy_render, lighting  # noqa: E402

HBM = 3.35e12
SMS, CLK = 132, 1.98e9
SFU_OPS = SMS * 16 * CLK


class Cam(types.SimpleNamespace):
    def __len__(self):
        return self.extrinsics.R.shape[0]


def timed(fn, min_s):
    fn(); torch.cuda.synchronize()
    t0 = time.perf_counter(); fn(); torch.cuda.synchronize()
    reps = max(3, int(min_s / max(time.perf_counter() - t0, 1e-6)))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def cost(P, C, L, phase, pixel_grads):
    """(bytes, sfu ops) for P pixels of which C are covered.  Forward: face_idx 8 B per pixel; normal,
    albedo, spec albedo, roughness 40 B per covered pixel; three images 36 B per pixel.  Backward: the
    same inputs and three image gradients (36 B per covered pixel) read, plus grad albedo, spec albedo,
    roughness and normals (40 B per pixel) when per-pixel gradients are requested.  Per (covered pixel,
    light): 8 SFU ops forward (two SG pairs), three times that backward."""
    if phase == "fwd":
        return 8 * P + 40 * C + 36 * P, C * L * 8
    return 8 * P + 76 * C + (40 * P if pixel_grads else 0), C * L * 24


def camera(B, res, dev):
    eye = torch.tensor([1.3, 0.9, 2.1], dtype=torch.float64)
    fwd = torch.nn.functional.normalize(-eye, dim=0)
    right = torch.nn.functional.normalize(torch.linalg.cross(fwd, torch.tensor([0., 1., 0.], dtype=torch.float64)), dim=0)
    up = torch.linalg.cross(right, fwd)
    R = torch.stack([right, up, -fwd]).float()
    f = res / 2 / math.tan(math.pi * 40 / 360)
    t = lambda v: torch.full((B,), v, device=dev)
    return Cam(extrinsics=types.SimpleNamespace(R=R[None].repeat(B, 1, 1).to(dev)), x0=t(3.5), y0=t(-2.25),
               focal_x=t(f), focal_y=t(f), width=res, height=res)


def gbuffer(cam, B, H, W, dev, gen):
    view = OSH.view_dirs(cam.extrinsics.R.double().cpu(), cam.x0.double().cpu(), cam.y0.double().cpu(),
                         cam.focal_x.double().cpu(), cam.focal_y.double().cpu(), cam.width, cam.height, H, W)
    view = view.float().to(dev)
    rnd = lambda *s: torch.rand(s, device=dev, generator=gen)
    yy, xx = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    r = 0.35 + 0.1 * torch.arange(B, device=dev)[:, None, None] / B
    inside = ((xx / W - 0.5) ** 2 + (yy / H - 0.5) ** 2) < r * r
    face_idx = torch.where(inside, (rnd(B, H, W) * 20000).long(), -1)
    t = torch.nn.functional.normalize(torch.randn((B, H, W, 3), device=dev, generator=gen), dim=-1)
    t = torch.nn.functional.normalize(t - (t * view).sum(-1, keepdim=True) * view, dim=-1)
    c = 0.25 + 0.75 * rnd(B, H, W, 1)
    normals = c * view + torch.sqrt(1 - c * c) * t
    del t
    base, metal = rnd(B, H, W, 3), rnd(B, H, W, 1)
    return face_idx, [base * (1 - metal), (1 - metal) * 0.04 + base * metal, 0.3 + 0.7 * rnd(B, H, W, 1), normals], view


def composed(view):
    def fn(cam, face_idx, albedo, spec_albedo, roughness, normals, amp, dirs, sharp):
        mask = face_idx >= 0
        n = torch.nn.functional.normalize(normals[mask], dim=-1)
        d = lighting.sg_diffuse_inner_product(amp, dirs, sharp, n, albedo[mask])
        s = lighting.sg_warp_specular_term(amp, dirs, sharp, n, roughness[mask].reshape(-1), view[mask],
                                           spec_albedo[mask])
        z = torch.zeros(face_idx.shape + (3,), device=albedo.device)
        return z.index_put((mask,), d), z.index_put((mask,), s), z.index_put((mask,), d + s)
    return fn


def torch32(view):
    return lambda cam, f, *a: OSH.sg_shade(view, f, *a)


def check(cam, face_idx, maps, lights, ws, view):
    """Errors of ours and of the fp32 formulation relative to the fp64 one's scale, on view 0."""
    f0 = face_idx[:1]
    m0 = [t[:1] for t in maps]
    w0 = [w[:1] for w in ws]
    cam0 = Cam(extrinsics=types.SimpleNamespace(R=cam.extrinsics.R[:1]), x0=cam.x0[:1], y0=cam.y0[:1],
               focal_x=cam.focal_x[:1], focal_y=cam.focal_y[:1], width=cam.width, height=cam.height)
    names = ("diffuse", "specular", "img", "g_albedo", "g_spec_albedo", "g_roughness", "g_normals",
             "g_amp", "g_dir", "g_sharp")

    def run(fn, ins, wts):
        leaves = [t.detach().clone().requires_grad_(True) for t in ins]
        outs = fn(cam0, f0, *leaves)
        sum((o * w).sum() for o, w in zip(outs, wts)).backward()
        return [o.detach() for o in outs] + [t.grad for t in leaves]
    mine = run(easy_render.sg_shade, m0 + list(lights), w0)
    r64 = run(lambda c, f, *a: OSH.sg_shade(view[:1].double(), f, *a), [t.double() for t in m0 + list(lights)],
              [w.double() for w in w0])
    r32 = run(lambda c, f, *a: OSH.sg_shade(view[:1], f, *a), m0 + list(lights), w0)
    err, err32 = {}, {}
    for k, a, b, c in zip(names, mine, r64, r32):
        scale = max(float(b.abs().max()), 1e-30)
        err[f"err_{k}"] = float((a.double() - b).abs().max()) / scale
        err32[f"torch32_err_{k}"] = float((c.double() - b).abs().max()) / scale
    return err, err32


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--res", type=int, default=1024)
    ap.add_argument("--lights", default="1,8,32,128")
    ap.add_argument("--min-seconds", type=float, default=0.5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_shade.py measures on a CUDA device"
    dev = torch.device("cuda")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"device: {torch.cuda.get_device_name(0)}; nvidia-smi: {q}")
    gen = torch.Generator(device=dev); gen.manual_seed(0)
    B, H, W = args.views, args.res, args.res
    cam = camera(B, args.res, dev)
    face_idx, maps, view = gbuffer(cam, B, H, W, dev, gen)
    P, C = face_idx.numel(), int((face_idx >= 0).sum())
    ws = [torch.rand((B, H, W, 3), device=dev, generator=gen) - 0.3 for _ in range(3)]
    paths = {"ours": easy_render.sg_shade, "composed": composed(view), "torch": torch32(view)}
    rows = []
    for L in [int(x) for x in args.lights.split(",")]:
        amp = torch.rand((L, 3), device=dev, generator=gen) * 2
        d = torch.nn.functional.normalize(torch.randn((L, 3), device=dev, generator=gen), dim=-1)
        s = torch.exp(torch.rand((L,), device=dev, generator=gen) * math.log(100.)) * 0.5
        row = {"L": L, "views": B, "res": args.res, "coverage": round(C / P, 4)}
        for impl, fn in paths.items():
            lp = [t.clone().requires_grad_(True) for t in (amp, d, s)]
            mp = [t.clone().requires_grad_(True) for t in maps]
            loss = lambda outs: sum((o * w).sum() for o, w in zip(outs, ws))
            try:
                with torch.no_grad():
                    row[f"{impl}_fwd_ms"] = timed(lambda: fn(cam, face_idx, *maps, *lp), args.min_seconds)
                row[f"{impl}_fwdbwd_all_ms"] = timed(lambda: loss(fn(cam, face_idx, *mp, *lp)).backward(),
                                                     args.min_seconds)
                row[f"{impl}_fwdbwd_lights_ms"] = timed(lambda: loss(fn(cam, face_idx, *maps, *lp)).backward(),
                                                        args.min_seconds)
            except torch.OutOfMemoryError:
                row[f"{impl}_fwd_ms"] = "out of memory"
            del lp, mp
            torch.cuda.empty_cache()
        errs, errs32 = check(cam, face_idx, maps, (amp, d, s), ws, view)
        row.update(errs)
        row.update(errs32)
        bad = {k: v for k, v in errs.items() if v > max(1e-5, 4 * errs32["torch32_" + k])}
        assert not bad, (L, bad)
        for phase, key, pg in (("fwd", "ours_fwd_ms", False), ("bwd", "ours_fwdbwd_all_ms", True),
                               ("bwd", "ours_fwdbwd_lights_ms", False)):
            byt, sfu = cost(P, C, L, phase, pg)
            if phase == "bwd":
                b2, s2 = cost(P, C, L, "fwd", False)
                byt, sfu = byt + b2, sfu + s2
            bound = max(("HBM", byt / HBM), ("SFU", sfu / SFU_OPS), key=lambda x: x[1])
            row[key.replace("_ms", "_bound")] = bound[0]
            row[key.replace("_ms", "_frac")] = round(bound[1] * 1e3 / row[key], 3)
        rows.append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"bench": "shade", "device": torch.cuda.get_device_name(0), "nvidia_smi": q, "rows": rows}))


if __name__ == "__main__":
    main()
