"""Times voxelgrids_to_trianglemeshes (csrc/marching_cubes.cu) on one GPU at sides 64, 128, 200 and 256,
B = 1 and 8, on three inputs: a uint8 binary sphere, a float occupancy field (a smooth ball plus
noise), and the same float field requiring grad.  Reports the forward and, for the input with grad,
the forward + backward; and the reference's operator (oracle/_ref, when it has been built) through
the reference wrapper's per-view steps (float copy, pad, torch.all, the operator, .long()), on the
same GPU.  Each reference output is checked equal to ours where the reference is correct, and marked
"truncated" where its launch drops voxels (sides 4, 5 and >= 202) or its vertex cap cuts the mesh.
A byte model computed from the shapes gives the forward's share of HBM bandwidth.  Prints the device,
its power limit, a table, and one JSON line.

    python scripts/bench_marching_cubes.py [--sizes 64 128 200 256] [--batch 1 8] [--iters 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
from kaolin_b200.ops import conversions  # noqa: E402
from oracle import build_ref_mcube  # noqa: E402

DEV = "cuda"
HBM_GBS = 3350.0      # H100 SXM5 HBM3 peak


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def grids(kind, n, B):
    x = torch.linspace(-1, 1, n, device=DEV)
    out = []
    for b in range(B):
        c = 0.1 * (b % 4) - 0.15
        d = torch.sqrt((x[:, None, None] - c) ** 2 + (x[None, :, None] + c) ** 2 + x[None, None, :] ** 2)
        if kind == "u8 sphere":
            out.append((d < 0.6 + 0.05 * b).to(torch.uint8))
        else:
            gen = torch.Generator(device=DEV).manual_seed(b)
            out.append((1.1 - d + 0.1 * torch.randn((n, n, n), device=DEV, generator=gen)).clamp(0, 1))
    return torch.stack(out)


def forward_bytes(B, n, elem, nv, nf):
    """Bytes the forward moves, from shapes: the input read once (its eight corner reads hit L1/L2),
    per cube 1 byte of case and 8 of counts written, the two scans (counts read twice, scans written
    once: 24 bytes), the emit pass's scan read (4 bytes), and the vertices and faces written."""
    cubes = B * (n + 2) ** 3
    return B * n ** 3 * elem + cubes * (1 + 8 + 24 + 4) + 12 * nv + 24 * nf


def reference_wrapper(mod, voxelgrids, iso=0.5):
    vg = F.pad(voxelgrids.float(), (1, 1, 1, 1, 1, 1), "constant", 0)
    verts, faces = [], []
    for i in range(vg.shape[0]):
        cur = vg[i]
        if torch.all(cur == 0):
            verts.append(torch.zeros((0, 3), device=DEV))
            faces.append(torch.zeros((0, 3), dtype=torch.long, device=DEV))
            continue
        v, f = mod.unbatched_mcube_forward_cuda(cur, iso)
        verts.append(v)
        faces.append(f.long())
    return verts, faces


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[64, 128, 200, 256])
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    name = torch.cuda.get_device_name()
    try:       # the device torch runs on, by UUID (CUDA_VISIBLE_DEVICES renumbers the indices)
        uuid = f"GPU-{torch.cuda.get_device_properties(torch.cuda.current_device()).uuid}"
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", uuid],
                               capture_output=True, text=True, timeout=30).stdout.strip() or "unknown"
    except Exception:
        power = "unknown"
    print(f"device: {name}, power limit: {power}")
    ref = build_ref_mcube.load()
    mc = conversions.voxelgrids_to_trianglemeshes
    rows = []
    print(f"{'n':>4} {'B':>2} {'input':<14} {'nv':>10} {'fwd ms':>8} {'HBM %':>6} {'f+b ms':>8} {'ref ms':>9} check")
    for n in args.sizes:
        for B in args.batch:
            for kind in ("u8 sphere", "f32 occupancy", "f32 with grad"):
                g = grids(kind, n, B)
                row = dict(n=n, B=B, input=kind)
                if kind == "f32 with grad":
                    g.requires_grad_(True)

                    def step():
                        verts, _ = mc(g)
                        torch.cat(verts).sum().backward()
                    row["fwd_bwd_ms"] = timed(step, args.iters)
                    g.grad = None
                with torch.no_grad():
                    verts, faces = mc(g)
                    row["fwd_ms"] = timed(lambda: mc(g), args.iters)
                nv, nf = sum(len(v) for v in verts), sum(len(f) for f in faces)
                row["nv"], row["nf"] = nv, nf
                row["hbm_share"] = forward_bytes(B, n, g.element_size(), nv, nf) / (row["fwd_ms"] * 1e-3) / (HBM_GBS * 1e9)
                check = "-"
                if ref is not None and kind != "f32 with grad":
                    with torch.no_grad():
                        row["ref_ms"] = timed(lambda: reference_wrapper(ref, g), max(1, args.iters // 5))
                        rv, rf = reference_wrapper(ref, g)
                    cap = (n + 2) ** 2 * 100 - 3
                    if n in (4, 5) or n >= 202 or any(len(v) > cap for v in verts):
                        check = "truncated"
                    else:
                        ok = all(torch.equal(a, b) and torch.equal(c, d) for a, b, c, d in zip(verts, rv, faces, rf))
                        check = "equal" if ok else "DIFFERS"
                row["check"] = check
                rows.append(row)
                fb = f"{row['fwd_bwd_ms']:8.3f}" if "fwd_bwd_ms" in row else f"{'':>8}"
                rm = f"{row['ref_ms']:9.2f}" if "ref_ms" in row else f"{'-':>9}"
                print(f"{n:>4} {B:>2} {kind:<14} {nv:>10} {row['fwd_ms']:8.3f} {100 * row['hbm_share']:6.1f} {fb} {rm} "
                      f"{check}", flush=True)
                del g, verts, faces
                torch.cuda.empty_cache()
    print(json.dumps({"device": name, "power_limit": power, "rows": rows}))


if __name__ == "__main__":
    main()
