"""Time kaolin.ops.conversions.voxelgrids_to_cubic_meshes (is_trimesh=True) on the GPU against a torch
restatement of the reference's structure on the same GPU: a float conv3d giving every lattice point's
three voxel differences, torch.nonzero over it, then per view a boolean gather of the quads' corners
and torch.unique(dim=0) over them.  Outputs are checked equal; the baseline is skipped where it runs
out of memory.  The card's name and power limit are read in the same run.

Workloads: B in {1, 8} at n in {64, 128, 256} for a uint8 ball, an icosphere voxelized by this
library's trianglemeshes_to_voxelgrids (a thin shell, so about twice the faces of the ball) and a
50 %-density random float32 grid (about 1.5 faces per lattice point, the worst case for output).
Times are the median and range of CUDA-event-timed calls after warm-up, host read included.

"GB" models the traffic the call needs at least: the grid read once; the seven bit planes (7 bits per
lattice point) written by the count kernel and read by the emit kernel; 12 B per vertex and 48 B per
pair of triangles written.  The scan's traffic (1 B per lattice point) is left out.  "share" is that
over the call's time against the H100 SXM data sheet's 3.35 TB/s: an end-to-end rate, not a kernel's.

    python scripts/bench_cubic_meshes.py [--reps 10] [--sizes 64 128 256] [--batches 1 8] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kaolin_b200 import synthetic  # noqa: E402
from kaolin_b200.ops.conversions import trianglemeshes_to_voxelgrids, voxelgrids_to_cubic_meshes  # noqa: E402

DEV = torch.device("cuda:0")
PEAK_BW = 3.35e12


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as exc:
        return f"{torch.cuda.get_device_name(0)} (power limit unread: {exc})"


def timed(fn, reps, warmup=2):
    """Median and range (ms) of `reps` CUDA-event timings, after `warmup` calls."""
    for _ in range(warmup):
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


# The baseline: kernel a maps the padded grid to v(p) - v(p - e_a) at output index p + 1 - e_a.
_KERNELS = torch.zeros((3, 1, 2, 2, 2))
for _a in range(3):
    _KERNELS[_a, 0, 0, 0, 0] = -1
    _KERNELS[(_a, 0) + tuple(int(i == _a) for i in range(3))] = 1
_E = torch.eye(3)


def baseline(grids, is_trimesh=True):
    d = F.conv3d(grids.unsqueeze(1).float(), _KERNELS.to(grids.device), padding=1).round()   # (B, 3, X+1, Y+1, Z+1)
    axis, view, *q = torch.nonzero(d.transpose(0, 1), as_tuple=True)
    rev = d.transpose(0, 1)[(axis, view, *q)] == -1
    p = torch.stack(q, 1).float() - 1 + _E.to(d.device)[axis]
    eb, ec = _E.to(d.device)[(axis + 1) % 3], _E.to(d.device)[(axis + 2) % 3]
    quads = torch.stack([p, p + eb, p + eb + ec, p + ec], 1)                                 # (n, 4, 3)
    verts_out, faces_out = [], []
    for b in range(grids.shape[0]):
        mine = view == b
        corners = quads[mine].reshape(-1, 3)
        verts, inverse = torch.unique(corners, dim=0, return_inverse=True)
        faces = inverse.view(-1, 4)
        r = rev[mine]
        faces[r] = faces[r].flip(1)
        if is_trimesh:
            faces = torch.cat([faces[:, [0, 3, 1]], faces[:, [2, 1, 3]]])
        verts_out.append(verts)
        faces_out.append(faces)
    return verts_out, faces_out


def ball(B, n):
    c = torch.arange(n, device=DEV, dtype=torch.float32) - (n - 1) / 2
    r2 = c[:, None, None] ** 2 + c[None, :, None] ** 2 + c[None, None, :] ** 2
    return (r2 < (0.42 * n) ** 2).to(torch.uint8).expand(B, n, n, n).contiguous()


def icosphere(B, n):
    v, f = synthetic.icosphere(5)
    rng = np.random.default_rng(n + B)
    views = np.stack([v * rng.uniform(0.6, 1.0) + rng.normal(scale=0.1, size=3) for _ in range(B)])
    return trianglemeshes_to_voxelgrids(torch.from_numpy(views.astype(np.float32)).to(DEV),
                                        torch.from_numpy(f).to(DEV), n)


def random(B, n):
    g = torch.Generator(DEV).manual_seed(n + B)
    return (torch.rand((B, n, n, n), device=DEV, generator=g) < 0.5).float()


def model_bytes(grid, verts, faces):
    B, X, Y, Z = grid.shape
    lattice = B * (X + 1) * (Y + 1) * (Z + 1)
    nv = sum(v.shape[0] for v in verts)
    pairs = sum(f.shape[0] for f in faces) // 2
    return grid.numel() * grid.element_size() + 2 * lattice * 7 / 8 + 12 * nv + 48 * pairs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--base-reps", type=int, default=2)
    ap.add_argument("--sizes", type=int, nargs="+", default=[64, 128, 256])
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_cubic_meshes needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    print(f"card: {card()}")
    rows = []
    print("| workload | B | n | quads | vertices | ours ms (range) | baseline ms | speedup | GB | GB/s | share |")
    print("|---|---|---|---|---|---|---|---|---|---|---|")
    for kind, make in (("ball u8", ball), ("icosphere u8", icosphere), ("random f32", random)):
        for B in args.batches:
            for n in args.sizes:
                grid = make(B, n)
                torch.cuda.synchronize()
                verts, faces = voxelgrids_to_cubic_meshes(grid)
                med, lo, hi = timed(lambda: voxelgrids_to_cubic_meshes(grid), args.reps)
                row = dict(workload=kind, B=B, n=n, quads=sum(f.shape[0] for f in faces) // 2,
                           vertices=sum(v.shape[0] for v in verts), ms=med, ms_min=lo, ms_max=hi)
                row["gb"] = model_bytes(grid, verts, faces) / 1e9
                row["gbps"] = row["gb"] / (med / 1e3)
                row["share"] = row["gbps"] * 1e9 / PEAK_BW
                try:
                    bv, bf = baseline(grid)
                    row["equal"] = all(torch.equal(a, b) for a, b in zip(verts + faces, bv + bf))
                    del bv, bf
                    row["base_ms"] = timed(lambda: baseline(grid), args.base_reps, warmup=0)[0]
                except torch.cuda.OutOfMemoryError:
                    row["base_ms"], row["equal"] = None, None
                del verts, faces
                torch.cuda.empty_cache()
                rows.append(row)
                base = "OOM" if row["base_ms"] is None else f"{row['base_ms']:.1f}"
                speed = "" if row["base_ms"] is None else f"{row['base_ms'] / med:.0f}x"
                print(f"| {kind} | {B} | {n} | {row['quads']:,} | {row['vertices']:,} | {med:.2f} ({lo:.2f}-{hi:.2f}) "
                      f"| {base} | {speed} | {row['gb']:.2f} | {row['gbps']:.0f} | {100 * row['share']:.0f} % |",
                      flush=True)
                if row["equal"] is False:
                    sys.exit(f"outputs differ from the baseline: {kind} B={B} n={n}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(dict(card=card(), rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
