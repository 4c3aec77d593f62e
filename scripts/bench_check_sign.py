"""Times check_sign (csrc/check_sign.cu) on one GPU: noisy icospheres of levels 5-8 (20 480 to 1.31 M
faces), N = 10^5 and 10^6 points drawn uniformly in the mesh's box (the Simplicits and occupancy-sampling
workload), B = 1 and 8 (a differently jittered mesh per view).  Reports the build (CheckSign
construction, its one device-to-host read included), the query (S(points)), the mean number of
candidate faces a point is tested against (its cell's list plus the wide list, from a host restatement
of the binning of view 0), and the reference's operator (oracle/_ref, built by
oracle/build_ref_check_sign.py) driven as the reference's check_sign.py drives it, on the same GPU.
The surface is smooth: each vertex moves radially by up to a fifth of the edge length.  The
reference tests every (point, face) pair; its leg is skipped above REF_MAX_PAIRS pair tests, and
the table says so.  Where it runs, its result is checked equal to ours.  Prints the device, its power
limit, a table, and one JSON line.

    python scripts/bench_check_sign.py [--levels 5 6 7 8] [--points 100000 1000000] [--batch 1 8]
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
from kaolin_b200.ops.mesh import CheckSign  # noqa: E402
from oracle import build_ref_check_sign  # noqa: E402
from oracle import check_sign as O  # noqa: E402

DEV = "cuda"
REF_MAX_PAIRS = 2e10      # B * N * F above which the reference's O(N F) leg is not run


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


def mean_candidates(verts, faces, points):
    """Host restatement of check_sign.cu's binning of one view (float32 cell arithmetic): the mean over
    the points of (faces in the point's cell + faces on the wide list)."""
    f32 = np.float32
    m = np.array([np.ptp(verts[:, a]) for a in range(3)], verts.dtype).max()
    tri = (verts / m)[faces][:, :, 1:]
    lo, hi = tri.min(1).astype(f32), tri.max(1).astype(f32)
    F = len(faces)
    G = O.grid_side(F)
    a0, a1 = lo.min(0), hi.max(0)
    inv = (f32(G) / np.maximum(a1 - a0, f32(1e-20))).astype(f32)
    cell = lambda v: np.clip(((v.astype(f32) - a0) * inv).astype(f32), 0, G - 1).astype(np.int64)
    c0, c1 = cell(lo), cell(hi)
    n = (c1 - c0 + 1).prod(1)
    wide = int((n > O.CAP).sum())
    cnt = np.zeros((G, G), np.int64)
    keep = n <= O.CAP
    for dy in range(O.CAP):
        for dz in range(O.CAP):
            sel = keep & (c0[:, 0] + dy <= c1[:, 0]) & (c0[:, 1] + dz <= c1[:, 1])
            np.add.at(cnt, (c0[sel, 0] + dy, c0[sel, 1] + dz), 1)
    pc = cell((points[:, 1:] / m))
    return float(cnt[pc[:, 0], pc[:, 1]].mean()) + wide, G, wide


def reference_check_sign(ref, verts, faces, points):
    """check_sign.py:138-155 on the reference's operator."""
    lens = [verts[..., a].max(-1)[0] - verts[..., a].min(-1)[0] for a in range(3)]
    maxlen = torch.max(torch.stack(lens), 0)[0]
    verts, points = verts / maxlen.view(-1, 1, 1), points / maxlen.view(-1, 1, 1)
    out = []
    for b in range(verts.shape[0]):
        v = [torch.index_select(verts[b], 0, faces[:, k]).contiguous() for k in range(3)]
        out.append(ref.unbatched_mesh_intersection_cuda(points[b].contiguous(), *v) % 2 == 1.)
    return torch.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", type=int, nargs="+", default=[5, 6, 7, 8])
    ap.add_argument("--points", type=int, nargs="+", default=[100_000, 1_000_000])
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
    ref = build_ref_check_sign.load()
    print(f"reference operator: {'oracle/_ref loaded' if ref is not None else 'NOT BUILT (reference leg skipped)'}; "
          f"its leg runs up to {REF_MAX_PAIRS:.0e} pair tests")
    results = []
    for level in args.levels:
        v0, f = synthetic.icosphere(level)
        F = len(f)
        faces = torch.from_numpy(f).to(DEV)
        for B in args.batch:
            rng = np.random.default_rng(level * 10 + B)
            # radial noise of a fifth of the edge length (about 1 / 2^level): a smooth surface per view
            vs = np.stack([v0 * (1.0 + 0.2 / 2 ** level * rng.uniform(-1, 1, size=(len(v0), 1))) for _ in range(B)])
            verts = torch.from_numpy(vs.astype(np.float32)).to(DEV)
            r_build = timed(lambda: CheckSign(verts, faces), max(2, args.iters // 2))
            S = CheckSign(verts, faces)
            for N in args.points:
                pts = np.stack([O._uniform(rng, vs[b], N, 0.0) for b in range(B)]).astype(np.float32)
                points = torch.from_numpy(pts).to(DEV)
                r = dict(level=level, F=F, B=B, N=N, build_ms=r_build)
                r["query_ms"] = timed(lambda: S(points), args.iters)
                r["Gpoints_per_s"] = B * N / (r["query_ms"] * 1e-3) / 1e9
                cand, G, wide = mean_candidates(vs[0].astype(np.float32), f, pts[0])
                r.update(G=G, wide_faces=wide, mean_candidates=cand)
                pairs = B * N * F
                if ref is not None and pairs <= REF_MAX_PAIRS:
                    r["ref_ms"] = timed(lambda: reference_check_sign(ref, verts, faces, points), 1)
                    r["speedup_query"] = r["ref_ms"] / r["query_ms"]
                    r["speedup_build_query"] = r["ref_ms"] / (r["query_ms"] + r_build)
                    r["equal_to_reference"] = bool(torch.equal(reference_check_sign(ref, verts, faces, points),
                                                               S(points)))
                    assert r["equal_to_reference"], r
                else:
                    r["ref_ms"] = None
                    r["ref_skipped"] = f"{pairs:.1e} pair tests > {REF_MAX_PAIRS:.0e}" if ref is not None else "not built"
                r["inside_fraction"] = float(S(points).float().mean())
                results.append(r)
                ref_s = (f"ref {r['ref_ms']:.1f} ms, x{r['speedup_query']:.0f} query, "
                         f"x{r['speedup_build_query']:.0f} build+query, equal" if r["ref_ms"] is not None
                         else f"ref skipped ({r['ref_skipped']})")
                print(f"level {level} F {F} B {B} N {N}: G {G} wide {wide} cand/pt {cand:.1f} | build "
                      f"{r_build:.3f} ms, query {r['query_ms']:.3f} ms ({r['Gpoints_per_s']:.2f} Gpt/s) | {ref_s}",
                      flush=True)
                del points
            del S, verts
            torch.cuda.empty_cache()
    print(json.dumps(dict(device=name, power_limit=power, results=results)))


if __name__ == "__main__":
    main()
