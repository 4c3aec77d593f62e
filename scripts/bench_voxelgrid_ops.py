"""Time kaolin.ops.voxelgrid's fill, extract_surface, extract_odms and project_odms on the GPU against
the reference's own computations: for fill, scipy's binary_fill_holes per view on the host, including
the device-to-host copy ("not measured" where scipy is missing); for the other three, the reference's
torch expressions on the same GPU.  Outputs are checked equal.  The card's name and power limit are
read in the same run, and every case is timed in several rounds to show the spread.

"bytes" is the traffic the kernels need at least: the grid read once and the output written once,
plus, for fill, the int32 labels written by the first kernel and read by the last two.  "share" is
bytes over time against the H100 SXM data sheet's 3.35 TB/s.

    python scripts/bench_voxelgrid_ops.py [--quick] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kaolin_b200 import synthetic  # noqa: E402
from kaolin_b200.ops import voxelgrid as vg  # noqa: E402
from kaolin_b200.ops.conversions import trianglemeshes_to_voxelgrids  # noqa: E402

DEV = torch.device("cuda:0")
PEAK_BW = 3.35e12

try:
    from scipy import ndimage
except ImportError:      # the fill baseline is then "not measured"
    ndimage = None


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


def host_timed(fn, reps):
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        times.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(times)), float(min(times)), float(max(times))


# the reference's torch expressions (kaolin/ops/voxelgrid.py), on the same GPU
def ref_surface(g, mode):
    x = (g.half() if g.dtype == torch.bool else g).unsqueeze(1)
    if mode == "wide":
        return (F.avg_pool3d(x, 3, padding=1, stride=1).squeeze(1) < 1) * g.bool()
    return ((F.avg_pool3d(x, (3, 1, 1), padding=(1, 0, 0), stride=1).squeeze(1) < 1)
            | (F.avg_pool3d(x, (1, 3, 1), padding=(0, 1, 0), stride=1).squeeze(1) < 1)
            | (F.avg_pool3d(x, (1, 1, 3), padding=(0, 0, 1), stride=1).squeeze(1) < 1)) * g.bool()


def ref_odms(g):
    g = g.bool()
    dim = g.shape[-1]
    m = torch.cat([torch.arange(1, dim + 1, device=g.device), torch.arange(dim, 0, -1, device=g.device)])
    z = torch.max(g.unsqueeze(1) * m.view(1, 2, 1, 1, -1), dim=4)[0]
    y = torch.max(g.unsqueeze(1) * m.view(1, 2, 1, -1, 1), dim=3)[0]
    x = torch.max(g.unsqueeze(1) * m.view(1, 2, -1, 1, 1), dim=2)[0]
    return dim - torch.cat([z, y, x], dim=1)


def ref_project(odms, votes=1):
    B, dim = odms.shape[0], odms.shape[-1]
    grid = torch.ones((B, dim, dim, dim), dtype=torch.bool, device=odms.device)
    u = odms.clone().view(B, 3, 2, dim, dim)
    u[:, :, 0] = dim - u[:, :, 0]
    u = u.view(B, 6, dim, dim)
    i = torch.arange(dim, device=odms.device)
    s = ((i.view(1, 1, 1, -1) >= u[:, 0].unsqueeze(-1)).byte() + (i.view(1, 1, 1, -1) < u[:, 1].unsqueeze(-1)).byte()
         + (i.view(1, 1, -1, 1) >= u[:, 2].unsqueeze(-2)).byte() + (i.view(1, 1, -1, 1) < u[:, 3].unsqueeze(-2)).byte()
         + (i.view(1, -1, 1, 1) >= u[:, 4].unsqueeze(-3)).byte() + (i.view(1, -1, 1, 1) < u[:, 5].unsqueeze(-3)).byte())
    return (grid * votes - s) > 0


def scipy_fill(g):
    return torch.from_numpy(np.stack([ndimage.binary_fill_holes(v) for v in g.cpu().numpy()]))


def icosphere_grid(level, B, res, seed=1):
    v, f = synthetic.icosphere(level)
    rng = np.random.default_rng(seed)
    views = np.stack([v * rng.uniform(0.6, 1.0) + rng.normal(scale=0.1, size=3) for _ in range(B)])
    return trianglemeshes_to_voxelgrids(torch.from_numpy(views.astype(np.float32)).to(DEV),
                                        torch.from_numpy(f).to(DEV), res) != 0


def serpentine(n):
    g = torch.ones((n, n, n), dtype=torch.bool, device=DEV)
    rows = torch.arange(1, n - 1, 2, device=DEV)
    planes = torch.arange(1, n - 1, 2, device=DEV)
    turn_x = torch.where(torch.arange(len(rows) - 1, device=DEV) % 2 == 0, n - 2, 1)
    end = (n - 2 if (len(rows) - 1) % 2 == 0 else 1, int(rows[-1]))
    for p, z in enumerate(planes.tolist()):
        g[1:n - 1, rows, z] = False
        g[turn_x, rows[:-1] + 1, z] = False
        if p + 1 < len(planes):
            x, y = end if p % 2 == 0 else (1, 1)
            g[x, y, z + 1] = False
    g[0, 1, 1] = False
    return g[None]


def row(name, nbytes, ours, base, base_kind, equal):
    r = dict(case=name, ms=ours[0], ms_min=ours[1], ms_max=ours[2], bytes=nbytes,
             share=nbytes / (ours[0] * 1e-3) / PEAK_BW, baseline=base_kind, equal=equal)
    if base is None:
        r.update(base_ms=None, speedup=None)
    else:
        r.update(base_ms=base[0], base_ms_min=base[1], base_ms_max=base[2], speedup=base[0] / ours[0])
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--json")
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    reps = 3 if a.quick else a.reps
    rows = []
    gen = torch.Generator(DEV).manual_seed(0)

    def fill_case(name, g, host_reps=2):
        n = g.numel()
        ours = timed(lambda: vg.fill(g), reps)
        out = vg.fill(g)
        if ndimage is None:
            rows.append(row(name, 6 * n, ours, None, "scipy not installed: not measured", None))
            return
        base = host_timed(lambda: scipy_fill(g), host_reps)
        rows.append(row(name, 6 * n, ours, base, "scipy per view, host", bool(torch.equal(out.cpu(), scipy_fill(g)))))

    s = 128 if a.quick else 256
    fill_case(f"fill icosphere L6 8x{s}^3", icosphere_grid(6, 8, s))
    if not a.quick:
        fill_case("fill icosphere L6 1x512^3", icosphere_grid(6, 1, 512), 1)
        fill_case("fill icosphere L6 1x1024^3", icosphere_grid(6, 1, 1024), 1)
        fill_case("fill serpentine 1x512^3", serpentine(512), 1)
    fill_case(f"fill random 0.69 8x{s}^3", torch.rand((8, s, s, s), device=DEV, generator=gen) < 0.69, 1)

    shapes = [(8, s)] if a.quick else [(8, 256), (1, 512)]
    for B, n in shapes:
        g = torch.rand((B, n, n, n), device=DEV, generator=gen) < 0.69
        N = g.numel()
        tag = f"{B}x{n}^3"
        if B == 1:
            fill_case(f"fill random 0.69 {tag}", g, 1)
        for mode in ("wide", "thin"):
            ours = timed(lambda: vg.extract_surface(g, mode), reps)
            base = timed(lambda: ref_surface(g, mode), reps)
            eq = bool(torch.equal(vg.extract_surface(g, mode), ref_surface(g, mode)))
            rows.append(row(f"extract_surface {mode} bool {tag}", 2 * N, ours, base, "reference torch, GPU", eq))
        gf = torch.rand((B, n, n, n), device=DEV, generator=gen)
        ours = timed(lambda: vg.extract_surface(gf), reps)
        base = timed(lambda: ref_surface(gf, "wide"), reps)
        eq = bool(torch.equal(vg.extract_surface(gf), ref_surface(gf, "wide")))
        rows.append(row(f"extract_surface wide float32 {tag}", 5 * N, ours, base, "reference torch, GPU", eq))
        sparse = torch.rand((B, n, n, n), device=DEV, generator=gen) < 0.02
        ours = timed(lambda: vg.extract_odms(sparse), reps)
        base = timed(lambda: ref_odms(sparse), reps)
        odms = vg.extract_odms(sparse)
        eq = bool(torch.equal(odms, ref_odms(sparse)))
        rows.append(row(f"extract_odms bool {tag}", N + 48 * B * n * n, ours, base, "reference torch, GPU", eq))
        ours = timed(lambda: vg.project_odms(odms), reps)
        base = timed(lambda: ref_project(odms), reps)
        eq = bool(torch.equal(vg.project_odms(odms), ref_project(odms)))
        rows.append(row(f"project_odms int64 {tag}", N + 48 * B * n * n, ours, base, "reference torch, GPU", eq))

    head = card()
    print(f"# {head}")
    print(f"{'case':44s} {'ms (min-max)':>22s} {'GB':>7s} {'share':>6s} {'baseline ms':>12s} {'x':>8s}  equal")
    for r in rows:
        t = f"{r['ms']:.3f} ({r['ms_min']:.3f}-{r['ms_max']:.3f})"
        b = "not measured" if r["base_ms"] is None else f"{r['base_ms']:.2f}"
        x = "" if r["speedup"] is None else f"{r['speedup']:.1f}"
        print(f"{r['case']:44s} {t:>22s} {r['bytes'] / 1e9:7.3f} {100 * r['share']:5.1f}% {b:>12s} {x:>8s}  "
              f"{r['equal']}")
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(dict(card=head, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
