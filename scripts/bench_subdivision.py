"""Times Loop subdivision (csrc/mesh_topology.cu) on one GPU: coarse icosphere levels 3-5 with 1-3
iterations (level 5 with 3 iterations reaches c5's 1 310 720 faces), B = 1 and 32.  Reports the
build (LoopSubdivision construction), the apply forward and forward + backward, and the functional
subdivide_trianglemesh (build + apply); and, for the reference's structure, the torch restatement of
oracle/subdivision.py in fp32 on the same GPU, one view at a time as the reference must run, with its
levels prebuilt (its numpy build is not timed).  Every case checks 4096 sampled output rows against
fp64.  Prints the device, its power limit, a table, and one JSON line.

    python scripts/bench_subdivision.py [--levels 3 4 5] [--iterations 1 2 3] [--iters 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
from kaolin_b200 import synthetic  # noqa: E402
from kaolin_b200.ops import mesh  # noqa: E402
from oracle import subdivision as O  # noqa: E402

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


def torch_reference(levels, x):
    """The torch restatement, one view at a time."""
    outs = []
    for b in range(x.shape[0]):
        y = x[b:b + 1]
        for lv in levels:
            y, _ = O.apply_level(lv, y)
        outs.append(y)
    return torch.cat(outs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", type=int, nargs="+", default=[3, 4, 5])
    ap.add_argument("--iterations", type=int, nargs="+", default=[1, 2, 3])
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    print(f"device: {name}, power limit: {power}")
    results = []
    rng = np.random.default_rng(0)
    for level in args.levels:
        verts, f = synthetic.icosphere(level)
        V, faces_np = len(verts), np.asarray(f, np.int64)
        faces = torch.from_numpy(faces_np).to(DEV)
        for it in args.iterations:
            r = dict(level=level, iterations=it, V=V, F=len(faces_np), F_out=len(faces_np) * 4 ** it)
            r["build_ms"] = timed(lambda: mesh.LoopSubdivision(V, faces, it), args.iters)
            S = mesh.LoopSubdivision(V, faces, it)
            levels, Vl, fl = [], V, faces_np
            for _ in range(it):
                levels.append(O.level(Vl, fl))
                Vl, fl = Vl + len(levels[-1]["edges"]), levels[-1]["new_faces"]
            # bytes: each level's CSRs and edge records once, x read and y written per level
            csr = sum(4 * (3 * (lv["V"] + 1) + 3 * lv["F"] + 2 * len(lv["pairs"]) + 4 * len(lv["edges"])) + 8 * 3 * lv["F"]
                      for lv in levels)
            for B in (1, 32):
                x = (torch.from_numpy(np.asarray(verts, np.float32))[None]
                     * torch.from_numpy(1 + 0.1 * rng.uniform(size=(B, V, 1)).astype(np.float32))).to(DEV)
                xg = x.clone().requires_grad_(True)
                g = torch.randn((B, S.num_output_vertices, 3), device=DEV)
                r[f"B{B}_fwd_ms"] = timed(lambda: S(x), args.iters)
                r[f"B{B}_fwdbwd_ms"] = timed(lambda: S(xg).backward(g), args.iters)
                r[f"B{B}_function_ms"] = timed(lambda: mesh.subdivide_trianglemesh(x, faces, it), args.iters)
                xt = x.clone().requires_grad_(True)
                reps = max(1, args.iters // (4 if B > 1 else 1))
                r[f"B{B}_torch_fwd_ms"] = timed(lambda: torch_reference(levels, x), reps)
                r[f"B{B}_torch_fwdbwd_ms"] = timed(lambda: torch_reference(levels, xt).backward(g), reps)
                nbytes = csr + sum(4 * B * 3 * (lv["V"] + lv["V"] + len(lv["edges"])) for lv in levels)
                r[f"B{B}_fwd_MB"] = nbytes / 1e6
                r[f"B{B}_hbm_fraction"] = nbytes / (r[f"B{B}_fwd_ms"] * 1e-3) / (HBM_GBS * 1e9)
                # sampled rows of view 0 against fp64
                y = S(x)
                ref, _ = O.subdivide(x[:1].double(), faces_np, it)
                rows = torch.from_numpy(rng.choice(y.shape[1], min(y.shape[1], 4096), replace=False)).to(DEV)
                err = float((y[0, rows].double() - ref[0, rows]).abs().max()) / float(x.abs().max())
                r[f"B{B}_rel_err"] = err
                assert err <= 1e-6, (level, it, B, err)
                del x, xg, xt, g, y
            results.append(r)
            print(f"level {level} x{it}: F {r['F']} -> {r['F_out']} | build {r['build_ms']:.3f} ms | "
                  f"B1 fwd {r['B1_fwd_ms']:.3f} fwd+bwd {r['B1_fwdbwd_ms']:.3f} function {r['B1_function_ms']:.3f} "
                  f"torch {r['B1_torch_fwd_ms']:.3f} / {r['B1_torch_fwdbwd_ms']:.3f} | "
                  f"B32 fwd {r['B32_fwd_ms']:.3f} fwd+bwd {r['B32_fwdbwd_ms']:.3f} function {r['B32_function_ms']:.3f} "
                  f"torch {r['B32_torch_fwd_ms']:.3f} / {r['B32_torch_fwdbwd_ms']:.3f} | "
                  f"B32 fwd {r['B32_fwd_MB']:.1f} MB, {100 * r['B32_hbm_fraction']:.0f}% of HBM | "
                  f"rel err {max(r['B1_rel_err'], r['B32_rel_err']):.1e}", flush=True)
            torch.cuda.empty_cache()
    print(json.dumps(dict(device=name, power_limit=power, results=results)))


if __name__ == "__main__":
    main()
