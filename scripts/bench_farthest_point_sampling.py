"""Time kaolin.ops.pointcloud.farthest_point_sampling on the GPU against the contract's torch oracle
(oracle/pointcloud.py) on the same GPU, which is what a user without NVIDIA Warp would write.  The
reference's own sampler needs Warp and is not measured.  Outputs are checked equal.  The card's name
and power limit are read in the same run, every case is timed in several rounds (CUDA events) to
show the spread, and the path and cluster size each workload took are printed.

Workloads: the Simplicits RKPM setup (1024 nodes from 10^5 points, 10^4 samples from 10^6), one
large view whose points overflow the chip (2^22), a PointNet++-style batch (32 x 8192), and one view
just below and one just above the cluster-to-grid boundary.

    python scripts/bench_farthest_point_sampling.py [--reps 5] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kaolin_b200 import _lib  # noqa: E402
from kaolin_b200.ops import pointcloud as pc  # noqa: E402
from oracle import pointcloud as opc  # noqa: E402

DEV = torch.device("cuda:0")
PATHS = {_lib.FPS_CLUSTER: "cluster", _lib.FPS_GRID: "grid"}


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as exc:
        return f"{torch.cuda.get_device_name(0)} (power limit unread: {exc})"


def timed(fn, reps):
    """Median and range (ms) of `reps` CUDA-event timings, after one warm-up call."""
    fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        start.record()
        fn()
        end.record()
        end.synchronize()
        times.append(start.elapsed_time(end))
    return float(np.median(times)), float(min(times)), float(max(times))


def grid_boundary():
    """The smallest N that takes the grid path, from the workspace query."""
    lo, hi = 1, 1 << 22
    while lo < hi:
        mid = (lo + hi) // 2
        if _lib.farthest_point_sampling_workspace_bytes(1, mid, 1, DEV, "plan")[1] == _lib.FPS_GRID:
            hi = mid
        else:
            lo = mid + 1
    return lo


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--baseline-reps", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    g = grid_boundary()
    workloads = [
        ("Simplicits nodes", 1, 10 ** 5, 1024),
        ("Simplicits samples", 1, 10 ** 6, 10 ** 4),
        ("one view of 2^22", 1, 1 << 22, 1024),
        ("PointNet++ batch", 32, 8192, 1024),
        ("just below the grid boundary", 1, g - 1, 1024),
        ("just above the grid boundary", 1, g, 1024),
    ]
    print(f"card: {card()}")
    rows = []
    for name, B, N, k in workloads:
        gen = torch.Generator(device=DEV).manual_seed(N)
        points = torch.rand((B, N, 3), device=DEV, generator=gen)
        _, path, cluster = _lib.farthest_point_sampling_workspace_bytes(B, N, k, DEV, "plan")
        ours = pc.farthest_point_sampling(points, k)
        base = opc.farthest_point_sampling(points, k)
        equal = bool(torch.equal(ours, base))
        t = timed(lambda: pc.farthest_point_sampling(points, k), args.reps)
        tb = timed(lambda: opc.farthest_point_sampling(points, k), args.baseline_reps)
        row = dict(workload=name, B=B, N=N, k=k, path=PATHS[path], cluster=cluster, ms=t[0], ms_min=t[1],
                   ms_max=t[2], us_per_round=1e3 * t[0] / k, oracle_ms=tb[0], oracle_ms_min=tb[1],
                   oracle_ms_max=tb[2], speedup=tb[0] / t[0], equal=equal)
        rows.append(row)
        print(f"{name:30s} B={B:<3d} N={N:<8d} k={k:<6d} {PATHS[path]:7s} C={cluster:<2d} "
              f"{t[0]:9.3f} ms ({t[1]:.3f}-{t[2]:.3f})  {row['us_per_round']:7.2f} us/round  "
              f"oracle {tb[0]:10.2f} ms  x{row['speedup']:.1f}  equal={equal}", flush=True)
    print("reference (NVIDIA Warp): not measured, Warp is not installed")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card(), reps=args.reps, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
