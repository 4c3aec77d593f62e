"""Times marching tetrahedra and subdivide_tetmesh (csrc/mesh_topology.cu) on one GPU, on the
Freudenthal grid (synthetic.freudenthal_grid) at resolutions 32, 64 and 128 (128: 2.15 M vertices,
12.6 M tets) with a noisy sphere SDF, B = 1 and 8.  Reports the build (MarchingTetrahedra
construction), the call's forward and forward + backward (and its parts: the forward with inputs that
require grad, the concatenation of the views, the backward alone), the functional marching_tetrahedra
(build + call), and, for the reference's structure, oracle/marching_tets.marching_on_device in fp32:
the reference's per-view steps (valid-tet mask, unique over the valid tets' edges, boolean gathers),
each a torch op on the same GPU, one view at a time; its outputs are checked equal to ours.  Also
subdivide_tetmesh with 4 features, forward and forward + backward.  A byte model computed from the
shapes gives the forward's share of HBM bandwidth.  Every case checks 4096 sampled output vertices of
view 0 against fp64.  Prints the device, its power limit, a table, and one JSON line.

    python scripts/bench_marching_tets.py [--res 32 64 128] [--batch 1 8] [--iters 10]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
from kaolin_b200 import synthetic  # noqa: E402
from kaolin_b200.ops import conversions, mesh  # noqa: E402
from oracle import marching_tets as O  # noqa: E402

DEV = "cuda"
HBM_GBS = 3350.0      # H100 SXM5 HBM3 peak
GOLDEN = os.path.join(os.path.dirname(__file__), "..", "tests", "golden", "marching_tets.npz")


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


def forward_bytes(B, V, E, T, nv, nf):
    """Bytes the forward moves, from shapes: classify (tets and sdf per view, the edge list, the flags),
    the scan (flags read twice, written once), the vertex kernel (scan, edges, vid, x, the vertices),
    the face kernel (tets and sdf again, the scan, tet_edge and vid of the surface tets, the faces)."""
    per_view = 32 * T + 8 * E + 4 * V + 4 * (E + 2 * T)
    per_view += 12 * (E + 2 * T)
    per_view += 4 * E + 8 * E + 4 * E + 12 * V
    per_view += 32 * T + 4 * V + 8 * T
    return B * per_view + 12 * nv + 24 * nf + 36 * nf


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, nargs="+", default=[32, 64, 128])
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
    g = np.load(GOLDEN)
    table = O.case_table(g["single_0123_out_faces"], g["single_0123_nf"])
    table_dev = torch.from_numpy(table).to(DEV)
    results = []
    for res in args.res:
        verts, tets_np = synthetic.freudenthal_grid(res)
        V, T = len(verts), len(tets_np)
        tets = torch.from_numpy(tets_np).to(DEV)
        t0 = time.perf_counter()
        topo_np = O.topology(V, tets_np)
        np_build_s = time.perf_counter() - t0
        r = dict(res=res, V=V, T=T, E=len(topo_np[0]), oracle_numpy_build_s=np_build_s)
        r["build_ms"] = timed(lambda: conversions.MarchingTetrahedra(V, tets), max(2, args.iters // 2))
        M = conversions.MarchingTetrahedra(V, tets)
        E = M._topo.num_edges
        assert E == r["E"]
        for B in args.batch:
            gen = torch.Generator(device="cpu").manual_seed(res * 100 + B)
            x = (torch.from_numpy(verts)[None] + 0.004 * (torch.rand((B, V, 3), generator=gen) - 0.5)).to(DEV)
            s = (x.norm(dim=-1) - 0.3 + 0.02 * torch.randn((B, V), generator=gen).to(DEV)).contiguous()
            out = M(x, s)
            nv, nf = sum(len(o) for o in out[0]), sum(len(o) for o in out[1])
            xg, sg = x.clone().requires_grad_(True), s.clone().requires_grad_(True)
            gout = torch.randn((nv, 3), device=DEV)
            r[f"B{B}_nv"], r[f"B{B}_nf"] = nv, nf
            r[f"B{B}_fwd_ms"] = timed(lambda: M(x, s), args.iters)
            r[f"B{B}_fwdbwd_ms"] = timed(lambda: torch.cat(M(xg, sg)[0]).backward(gout), args.iters)
            # the parts of fwd+bwd: the forward with inputs that require grad (it records the graph), the
            # same plus the concatenation, and the backward alone through a graph kept alive
            r[f"B{B}_fwd_grad_ms"] = timed(lambda: M(xg, sg), args.iters)
            r[f"B{B}_fwd_grad_cat_ms"] = timed(lambda: torch.cat(M(xg, sg)[0]), args.iters)
            y = torch.cat(M(xg, sg)[0])
            r[f"B{B}_bwd_ms"] = timed(lambda: y.backward(gout, retain_graph=True), args.iters)
            del y
            r[f"B{B}_function_ms"] = timed(lambda: conversions.marching_tetrahedra(x, tets, s), max(2, args.iters // 2))
            # the reference's structure, every step a torch op on this GPU, one view at a time
            reps = 3 if res >= 128 else max(3, args.iters // 2)
            r[f"B{B}_torch_fwd_ms"] = timed(lambda: [O.marching_on_device(x[b:b + 1], tets, s[b:b + 1], table_dev)
                                                     for b in range(B)], reps)
            base = O.marching_on_device(x[:1], tets, s[:1], table_dev)[0]
            assert torch.equal(base[1], out[1][0]) and torch.equal(base[0], out[0][0])
            nbytes = forward_bytes(B, V, E, T, nv, nf)
            r[f"B{B}_fwd_MB"] = nbytes / 1e6
            r[f"B{B}_hbm_fraction"] = nbytes / (r[f"B{B}_fwd_ms"] * 1e-3) / (HBM_GBS * 1e9)
            # 4096 sampled vertices of view 0 against fp64 (same faces, exactly)
            ref = O.marching(x[:1].double(), tets_np, s[:1].double(), table, topo_np)[0]
            assert torch.equal(out[1][0].cpu(), ref[1])
            rows = torch.from_numpy(np.random.default_rng(res).choice(len(ref[0]), min(len(ref[0]), 4096),
                                                                      replace=False)).to(DEV)
            err = float((out[0][0][rows].double() - ref[0][rows]).abs().max()) / float(x.abs().max())
            r[f"B{B}_rel_err"] = err
            assert err <= 1e-6, (res, B, err)
            # subdivide_tetmesh with the sdf and 3 more features
            feats = torch.cat([s[..., None], x], -1)
            xs, fs = x.clone().requires_grad_(True), feats.clone().requires_grad_(True)
            r[f"B{B}_sub_fwd_ms"] = timed(lambda: mesh.subdivide_tetmesh(x, tets, feats), max(2, args.iters // 2))

            def sub_fb():
                y, _, yf = mesh.subdivide_tetmesh(xs, tets, fs)
                (y.sum() + yf.sum()).backward()
            r[f"B{B}_sub_fwdbwd_ms"] = timed(sub_fb, max(2, args.iters // 2))
            del x, s, xg, sg, gout, out, xs, fs, feats
            torch.cuda.empty_cache()
        results.append(r)
        line = f"res {res}: V {V} T {T} E {E} | build {r['build_ms']:.2f} ms"
        for B in args.batch:
            line += (f" | B{B} nf {r[f'B{B}_nf']} fwd {r[f'B{B}_fwd_ms']:.3f} fwd+bwd {r[f'B{B}_fwdbwd_ms']:.3f} "
                     f"(grad fwd {r[f'B{B}_fwd_grad_ms']:.3f}, +cat {r[f'B{B}_fwd_grad_cat_ms']:.3f}, "
                     f"bwd {r[f'B{B}_bwd_ms']:.3f}) "
                     f"function {r[f'B{B}_function_ms']:.2f} torch {r[f'B{B}_torch_fwd_ms']:.1f} ms, "
                     f"{r[f'B{B}_fwd_MB']:.0f} MB {100 * r[f'B{B}_hbm_fraction']:.0f}% HBM, "
                     f"sub {r[f'B{B}_sub_fwd_ms']:.2f}/{r[f'B{B}_sub_fwdbwd_ms']:.2f}, err {r[f'B{B}_rel_err']:.1e}")
        print(line, flush=True)
        del M, tets
        torch.cuda.empty_cache()
    print(json.dumps(dict(device=name, power_limit=power, results=results)))


if __name__ == "__main__":
    main()
