"""Host cost of one DIB-R forward + backward through the Python layer: ``_host.forward`` and
``_host.backward`` (argument handling, workspace, the library calls) at a size where the GPU work
is small - 1 view, 64x64, an icosphere, 3 feature channels.  Each round reports two times per pair:
- wall: ``--iters`` pairs enqueued and one synchronise at the end.  This is the larger of the host
  cost and the GPU time of a pair; the kernel time of one pair (the library's per-kernel trace) is
  printed beside it.
- enqueue: the host time inside the calls alone, the same number of pairs enqueued in bursts of
  ``BURST`` with a synchronise after each burst, so the launch queue never fills and blocks the host.
Prints the device, its power limit, every round, and one JSON line with the medians.

    python scripts/bench_host_call.py [--iters 1000] [--rounds 7]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
from kaolin_b200 import _lib, synthetic  # noqa: E402
from kaolin_b200.render.mesh import _host  # noqa: E402

SIGMAINV, BOXLEN, KNUM, MULT, EPS = 7000.0, 0.02, 30, 1000.0, 1e-8     # bench.py's DIB-R parameters
H = W = 64
BURST = 10          # pairs per burst: 100 launches, well inside the device's launch queue


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    print(f"device: {name}, power limit: {power}")

    dev = torch.device("cuda:0")
    fvz, fvi, fnz = synthetic.icosphere_views(1, 2, seed=0)
    ff = synthetic.random_features(1, fvz.shape[1], 3, seed=0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    fvz, fvi, fnz, ff = t(fvz), t(fvi), t(fnz), t(ff)
    g_feat = torch.rand((1, H, W, 3), device=dev)
    g_soft = torch.rand((1, H, W), device=dev)
    mode = _lib.RASTER | _lib.SOFT_MASK

    def step():
        _, idx, wts, soft, ws = _host.forward(mode, H, W, fvz, fvi, ff, fnz, None, MULT, EPS, SIGMAINV,
                                              BOXLEN * MULT, KNUM)
        _host.backward(H, W, g_feat, g_soft, idx, wts, soft, fvi, ff, MULT, EPS, SIGMAINV, BOXLEN * MULT,
                       KNUM, ws, True)

    for _ in range(50):
        step()
    torch.cuda.synchronize()
    _lib.trace_begin()
    step()
    kernels = _lib.trace_end()
    kernel_us = sum(ms for _, ms in kernels) * 1e3
    print(f"{fvz.shape[1]} faces; one pair runs {len(kernels)} kernels, {kernel_us:.1f} us of kernel time")
    wall_us, enqueue_us = [], []
    bursts = max(1, args.iters // BURST)
    for r in range(args.rounds):
        t0 = time.perf_counter()
        for _ in range(args.iters):
            step()
        torch.cuda.synchronize()
        wall_us.append((time.perf_counter() - t0) * 1e6 / args.iters)
        inside = 0.0
        for _ in range(bursts):
            t0 = time.perf_counter()
            for _ in range(BURST):
                step()
            inside += time.perf_counter() - t0
            torch.cuda.synchronize()
        enqueue_us.append(inside * 1e6 / (bursts * BURST))
        print(f"round {r}: wall {wall_us[-1]:.1f} us, enqueue {enqueue_us[-1]:.1f} us per forward + backward")
    print(json.dumps(dict(device=name, power_limit=power, faces=fvz.shape[1], iters=args.iters, rounds=args.rounds,
                          kernel_us=kernel_us, wall_us_median=statistics.median(wall_us),
                          enqueue_us_median=statistics.median(enqueue_us), enqueue_us_min=min(enqueue_us),
                          enqueue_us_max=max(enqueue_us))))


if __name__ == "__main__":
    main()
