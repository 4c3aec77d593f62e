"""Time trianglemeshes_to_voxelgrids and pointclouds_to_voxelgrids, dense and sparse, against the
reference's level-synchronous structure on the same GPU (oracle/voxelize.py: a Python loop over views,
one host read and boolean filter per subdivision level, the exact range prune on, and torch.unique once
at the end instead of once per level, which makes it faster than the reference itself).  Outputs are
checked equal.  The card's name and power limit are read in the same run.

Dense rows report the output-write bandwidth (the grid's bytes over the call's time) against the
H100 SXM data sheet's 3.35 TB/s.  "nodes" is the number of triangles the subdivision tests per call,
counted by the oracle on the same workload.

    python scripts/bench_voxelize.py [--quick] [--json out.json]
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

from kaolin_b200 import synthetic  # noqa: E402
from kaolin_b200.ops.conversions import pointclouds_to_voxelgrids, trianglemeshes_to_voxelgrids  # noqa: E402
from oracle import voxelize as ov  # noqa: E402

DEV = torch.device("cuda:0")
PEAK_BW = 3.35e12
CUBE_V = [[x, y, z] for x in (0., 1.) for y in (0., 1.) for z in (0., 1.)]
CUBE_F = [[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1],
          [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]]


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as exc:
        return f"{torch.cuda.get_device_name(0)} (power limit unread: {exc})"


def timed(fn, reps):
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
    return float(np.median(times))


def icosphere_views(level, B, seed=1):
    v0, f = synthetic.icosphere(level)
    rng = np.random.default_rng(seed)
    v = np.stack([v0 * (1 + 0.05 * rng.uniform(-1, 1, (v0.shape[0], 1))) for _ in range(B)]).astype(np.float32)
    return torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV)


def workloads(quick):
    cube = (torch.tensor(CUBE_V, device=DEV)[None], torch.tensor(CUBE_F, device=DEV))
    out = [(f"cube res {r}", cube, r, None, None) for r in (128, 256, 512)]
    for level in (5, 6):
        for B in (1, 8):
            mesh = icosphere_views(level, B)
            out += [(f"ico{level} B={B} res {r}", mesh, r, None, None) for r in (128, 256, 512)]
    v, f = icosphere_views(3, 1)
    out.append(("ico3 zoomed res 512", (v, f), 512, torch.tensor([[0.7, -0.2, -0.2]], device=DEV),
                torch.tensor([0.4], device=DEV)))
    g = torch.Generator(device=DEV).manual_seed(0)
    out.append(("points 1e6 B=8 res 256", (torch.randn((8, 10 ** 6, 3), generator=g, device=DEV), None), 256, None,
                None))
    return out[:3] + out[-2:] if quick else out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--json")
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    info = card()
    print(f"# {info}, torch {torch.__version__}")
    rows = []
    for name, (v, f), res, origin, scale in workloads(a.quick):
        if f is None:
            call = lambda sparse: pointclouds_to_voxelgrids(v, res, origin, scale, return_sparse=sparse)
        else:
            call = lambda sparse: trianglemeshes_to_voxelgrids(v, f, res, origin, scale, return_sparse=sparse)
        stats = {}

        def oracle():
            r = ov.voxel_rows(ov.normalize(v, origin, scale), res, f, prune=True, stats=stats)
            return ov.dense(r, v.shape[0], res, torch.float32), r

        t_dense = timed(lambda: call(False), a.reps)
        t_sparse = timed(lambda: call(True), a.reps)
        t_ref = timed(oracle, 2)
        dense, ref_rows = oracle()
        ok = torch.equal(call(True)._indices(), ref_rows.T) and torch.equal(call(False), dense)
        del dense
        nodes = stats.get("nodes", 0) // 3        # timed() ran the oracle three times
        out_bytes = v.shape[0] * res ** 3 * 4
        row = dict(workload=name, dense_ms=t_dense, sparse_ms=t_sparse, oracle_ms=t_ref,
                   speedup_dense=t_ref / t_dense, write_TBps=out_bytes / t_dense / 1e9,
                   write_share=out_bytes / t_dense / 1e-3 / PEAK_BW, nodes=nodes, voxels=int(ref_rows.shape[0]),
                   equal=bool(ok))
        rows.append(row)
        print(f"{name:26s} dense {t_dense:8.3f} ms  sparse {t_sparse:8.3f} ms  oracle {t_ref:9.2f} ms  "
              f"x{row['speedup_dense']:7.1f}  write {row['write_TBps']:5.2f} TB/s ({100 * row['write_share']:4.1f} %)  "
              f"nodes {nodes:>11d}  voxels {row['voxels']:>10d}  equal {ok}", flush=True)
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(dict(card=info, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
