"""Times point_to_mesh_distance (csrc/point_mesh_distance.cu) on one GPU: noisy icospheres of levels 3-6
(1280 to 81 920 faces), N = 2048 and 10^5 points near the surface, B = 1 and 8 (a differently jittered
mesh per view), forward alone and forward plus backward.  The reference's operator (oracle/_ref, built
by oracle/build_ref_point_mesh.py) runs on the same GPU the way its wrapper drives it: view by view,
zero-filled outputs, then torch.stack.  Its leg is skipped above REF_MAX_PAIRS pair evaluations, and the
table says so; where it runs, its dist, face_idx and dist_type are checked equal to ours.  Reports ms
and (point, face) pairs per second, prints the device and its power limit, a table and one JSON line.

    python scripts/bench_point_mesh_distance.py [--levels 3 4 5 6] [--points 2048 100000] [--batch 1 8]
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
from kaolin_b200.metrics import point_to_mesh_distance  # noqa: E402
from oracle import build_ref_point_mesh  # noqa: E402

DEV = "cuda"
REF_MAX_PAIRS = 3e10      # B * N * F above which the reference's leg is not run


def timed(fn, iters, warmup=3):
    for _ in range(warmup):   # the process's first autograd calls carry one-time host costs
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def workload(level, N, B, seed=0):
    rng = np.random.default_rng(seed)
    v, f = synthetic.icosphere(level)
    fv = []
    for _ in range(B):
        vb = v * (1 + 0.002 * rng.normal(size=(v.shape[0], 1)))
        fv.append(vb[f])
    d = rng.normal(size=(B, N, 3))
    d /= np.linalg.norm(d, axis=2, keepdims=True)
    p = d * (1 + 0.05 * rng.normal(size=(B, N, 1)))
    return (torch.from_numpy(p).float().to(DEV), torch.from_numpy(np.stack(fv)).float().to(DEV))


def ref_forward(ext, p, fv):
    dist, idx, typ = [], [], []
    for b in range(p.shape[0]):
        n = p.shape[1]
        d = torch.zeros((n,), device=DEV, dtype=p.dtype)
        i = torch.zeros((n,), device=DEV, dtype=torch.long)
        t = torch.zeros((n,), device=DEV, dtype=torch.int32)
        ext.unbatched_triangle_distance_forward_cuda(p[b], fv[b], d, i, t)
        dist.append(d); idx.append(i); typ.append(t)
    return torch.stack(dist), torch.stack(idx), torch.stack(typ)


def ref_forward_backward(ext, p, fv, g):
    _, idx, typ = ref_forward(ext, p, fv)
    for b in range(p.shape[0]):
        gp, gf = torch.zeros_like(p[b]), torch.zeros_like(fv[b])
        ext.unbatched_triangle_distance_backward_cuda(g[b], p[b], fv[b], idx[b], typ[b], gp, gf)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", type=int, nargs="+", default=[3, 4, 5, 6])
    ap.add_argument("--points", type=int, nargs="+", default=[2048, 100000])
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    ext = build_ref_point_mesh.load()
    name = torch.cuda.get_device_name(0)
    print(f"# {name}, power limit {power_limit()}")
    print(f"{'level':>5} {'F':>6} {'N':>7} {'B':>2} | {'fwd ms':>8} {'ref fwd':>8} {'x':>6} | {'f+b ms':>8} "
          f"{'ref f+b':>8} {'x':>6} | {'Gpairs/s':>8} {'ref':>8} | equal")
    rows = []
    for level in args.levels:
        for N in args.points:
            for B in args.batch:
                p, fv = workload(level, N, B)
                F = fv.shape[1]
                g = torch.randn(B, N, device=DEV)
                pr = p.clone().requires_grad_(True)
                fr = fv.clone().requires_grad_(True)

                def fwd():
                    return point_to_mesh_distance(p, fv)

                def fb():
                    d, _, _ = point_to_mesh_distance(pr, fr)
                    d.backward(g)

                iters = max(1, min(args.iters, int(2e11 / (B * N * F))))
                t_f, t_fb = timed(fwd, iters), timed(fb, iters)
                pairs = B * N * F
                row = {"level": level, "F": F, "N": N, "B": B, "fwd_ms": t_f, "fwd_bwd_ms": t_fb,
                       "pairs_per_s": pairs / (t_f * 1e-3), "ref_fwd_ms": None, "ref_fwd_bwd_ms": None,
                       "equal": None}
                if ext is not None and pairs <= REF_MAX_PAIRS:
                    ours = fwd()
                    ref = ref_forward(ext, p, fv)
                    row["equal"] = all(torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                                                   b.view(torch.int32) if b.dtype == torch.float32 else b)
                                       for a, b in zip(ours, ref))
                    row["ref_fwd_ms"] = timed(lambda: ref_forward(ext, p, fv), iters)
                    row["ref_fwd_bwd_ms"] = timed(lambda: ref_forward_backward(ext, p, fv, g), iters)
                rows.append(row)
                rf, rfb = row["ref_fwd_ms"], row["ref_fwd_bwd_ms"]
                fmt = lambda x: f"{x:8.3f}" if x is not None else "skipped".rjust(8)
                sp = lambda r, o: f"{r / o:6.1f}" if r is not None else "".rjust(6)
                rp = f"{pairs / (rf * 1e-3) / 1e9:8.1f}" if rf else "".rjust(8)
                print(f"{level:5d} {F:6d} {N:7d} {B:2d} | {t_f:8.3f} {fmt(rf)} {sp(rf, t_f)} | {t_fb:8.3f} "
                      f"{fmt(rfb)} {sp(rfb, t_fb)} | {row['pairs_per_s'] / 1e9:8.1f} {rp} | {row['equal']}",
                      flush=True)
    print(json.dumps({"device": name, "power_limit": power_limit(), "rows": rows}))


if __name__ == "__main__":
    main()
