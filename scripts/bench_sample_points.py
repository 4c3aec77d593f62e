"""Times surface sampling (csrc/sample_points.cu) on one GPU, forward alone and forward plus backward, for
three workloads: the DMTet step (B = 1, level-7 icosphere, 327 680 faces, N = 5e4), ShapeNet-style
preprocessing (B = 8, level 6, N = 1e5, UV features D = 2) and a large mesh (B = 1, level 8, 1 310 720
faces, N = 1e6).  Three legs run on the same GPU: ``SurfaceSampler`` (topology built once), the functional
``sample_points`` (a topology build and one status read per call when vertices need a gradient) and a
torch restatement of the reference's steps (index_select, the area expression, Categorical sampling,
gather, rand, interpolation; autograd backward), written from the reference's description.  Reports ms,
algorithmic bytes per second (vertex, face and feature reads plus output writes of one call), the
topology build time and the card's name and power limit, a table and one JSON line.

    python scripts/bench_sample_points.py [--iters 20]
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
from kaolin_b200.ops import mesh  # noqa: E402

DEV = "cuda"
WORKLOADS = [("dmtet", 1, 7, 50000, 0), ("preprocess", 8, 6, 100000, 2), ("large", 1, 8, 1000000, 0)]


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in out.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(), "unknown"]


def torch_reference(vertices, faces, num_samples, face_features=None):
    """The reference's steps in plain torch (trianglemesh.py:30-93, 159-240 as described there)."""
    fv = [torch.index_select(vertices, 1, faces[:, k]) for k in range(3)]
    x, y = fv[0] - fv[1], fv[1] - fv[2]
    a = (x[..., 1] * y[..., 2] - x[..., 2] * y[..., 1]) ** 2
    b = (x[..., 2] * y[..., 0] - x[..., 0] * y[..., 2]) ** 2
    c = (x[..., 0] * y[..., 1] - x[..., 1] * y[..., 0]) ** 2
    areas = torch.sqrt(a + b + c) * 0.5
    choices = torch.distributions.Categorical(areas).sample([num_samples]).transpose(0, 1)
    idx = choices[..., None].expand(-1, -1, 3)
    v = [torch.gather(f, 1, idx) for f in fv]
    u = torch.sqrt(torch.rand(choices.shape + (1,), device=vertices.device, dtype=vertices.dtype))
    w = torch.rand(choices.shape + (1,), device=vertices.device, dtype=vertices.dtype)
    w0, w1, w2 = 1 - u, u * (1 - w), u * w
    points = w0 * v[0] + w1 * v[1] + w2 * v[2]
    if face_features is None:
        return points, choices
    D = face_features.shape[-1]
    g = torch.gather(face_features, 1, choices[..., None, None].expand(-1, -1, 3, D))
    return points, choices, w0 * g[:, :, 0] + w1 * g[:, :, 1] + w2 * g[:, :, 2]


def bytes_moved(B, V, F, N, D, ts):
    """Vertices and faces read, areas and the float64 CDF written and read, samples written (+ features)."""
    return B * V * 3 * ts + F * 24 + B * F * (3 * 8 + 8) + B * N * (3 * ts + 8 + D * ts) + B * F * 3 * D * ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    name, power = card()
    print(f"device: {name}, power limit {power}")
    rows = []
    for label, B, level, N, D in WORKLOADS:
        v, f = synthetic.icosphere(level)
        rng = np.random.default_rng(level)
        v = np.stack([np.asarray(v) * (1 + 0.1 * b) + rng.normal(scale=0.003, size=np.shape(v)) for b in range(B)])
        vt = torch.tensor(v, dtype=torch.float32, device=DEV).requires_grad_(True)
        ft = torch.tensor(np.asarray(f), dtype=torch.int64, device=DEV)
        F, V = ft.shape[0], vt.shape[1]
        ff = torch.randn((B, F, 3, D), device=DEV, requires_grad=True) if D else None

        torch.cuda.synchronize()
        t0 = time.perf_counter()
        S = mesh.SurfaceSampler(V, ft)
        torch.cuda.synchronize()
        build_ms = (time.perf_counter() - t0) * 1e3
        build_ms = min(build_ms, timed(lambda: mesh.SurfaceSampler(V, ft), 5, warmup=1))

        def loss(out):
            return out[0].sum() + (out[2].sum() if D else 0)

        legs = {"sampler": lambda: S(vt, N, face_features=ff),
                "functional": lambda: mesh.sample_points(vt, ft, N, face_features=ff),
                "torch": lambda: torch_reference(vt, ft, N, ff)}
        res = {}
        for leg, fn in legs.items():
            with torch.no_grad():
                fwd = timed(fn, args.iters)
            both = timed(lambda: loss(fn()).backward(), args.iters)
            res[leg] = (fwd, both)
        moved = bytes_moved(B, V, F, N, D, 4)
        row = dict(workload=label, B=B, faces=F, N=N, D=D, topology_build_ms=round(build_ms, 3),
                   **{f"{leg}_fwd_ms": round(r[0], 4) for leg, r in res.items()},
                   **{f"{leg}_fwd_bwd_ms": round(r[1], 4) for leg, r in res.items()},
                   sampler_fwd_GBps=round(moved / res["sampler"][0] / 1e6, 1),
                   speedup_fwd_vs_torch=round(res["torch"][0] / res["sampler"][0], 2),
                   speedup_fwd_bwd_vs_torch=round(res["torch"][1] / res["sampler"][1], 2))
        rows.append(row)
        print(f"{label:11s} B={B} F={F:8d} N={N:8d} D={D} | build {build_ms:7.3f} ms | "
              + " | ".join(f"{leg} {r[0]:7.3f}/{r[1]:7.3f} ms" for leg, r in res.items())
              + f" | sampler fwd {row['sampler_fwd_GBps']} GB/s")
    print(json.dumps(dict(device=name, power_limit=power, rows=rows)))


if __name__ == "__main__":
    main()
