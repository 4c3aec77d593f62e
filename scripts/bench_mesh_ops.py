"""Times the mesh Laplacian and vertex averaging (csrc/mesh_topology.cu) on icosphere levels 5-8 on one
GPU, against the reference's dense path (where it fits), torch.sparse.mm on a CSR tensor of the same
indices, and the reference's scatter_add_ chain for averaging.  Every output is checked against the
fp64 oracle on a sample of rows.  Prints the device, its power limit, a table, and one JSON line.

    python scripts/bench_mesh_ops.py [--levels 5 6 7 8] [--iters 20]
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
from kaolin_b200.metrics.trianglemesh import uniform_laplacian_smoothing  # noqa: E402
from kaolin_b200.ops import mesh  # noqa: E402

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


def try_time(fn, iters):
    try:
        return timed(fn, iters)
    except torch.OutOfMemoryError:
        torch.cuda.empty_cache()
        return None


def ref_dense_laplacian(V, faces):
    """The reference's uniform_laplacian (kaolin/ops/mesh/mesh.py:116-151), restated in torch."""
    fi = torch.stack([faces, torch.roll(faces, 1, dims=-1)], dim=-1)
    bi = torch.stack([torch.roll(faces, 1, dims=-1), faces], dim=-1)
    idx = torch.cat([fi, bi], dim=1).reshape(-1, 2).unique(dim=0)
    A = torch.zeros((V, V), device=faces.device)
    A[idx[:, 0], idx[:, 1]] = 1
    L = A / A.sum(1).view(-1, 1)
    torch.diagonal(L)[:] = -1
    L[torch.isnan(L)] = 0
    return L


def ref_average(faces, ff, V):
    B, F, S, N = ff.shape
    out = torch.zeros((B, V, N), device=ff.device)
    cnt = torch.zeros((B, V), device=ff.device)
    fr = faces.unsqueeze(0).repeat(B, 1, 1)
    ones = torch.ones((B, F), device=ff.device)
    for i in range(S):
        out.scatter_add_(1, fr[..., i:i + 1].repeat(1, 1, N), ff[..., i, :])
        cnt.scatter_add_(1, fr[..., i], ones)
    return out / cnt.clip(min=1).unsqueeze(-1)


def fmt(ms):
    return "out of memory" if ms is None else f"{ms:.3f}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", type=int, nargs="+", default=[5, 6, 7, 8])
    ap.add_argument("--iters", type=int, default=20)
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
        V, F = len(verts), len(f)
        faces = torch.from_numpy(np.asarray(f, np.int64)).to(DEV)
        r = dict(level=level, V=V, F=F)
        r["build_ms"] = timed(lambda: mesh.UniformLaplacian(V, faces), args.iters)
        L = mesh.UniformLaplacian(V, faces)
        topo = L._topo
        E = topo.num_edges
        csr = torch.sparse_csr_tensor(topo.adj_ptr.long(), topo.adj.long(),
                                      torch.repeat_interleave(topo.weight, topo.degree.long()), (V, V))
        for B in (1, 32):
            x = torch.from_numpy(rng.normal(size=(B, V, 3)).astype(np.float32)).to(DEV).requires_grad_(True)
            g = torch.randn((B, V, 3), device=DEV)
            r[f"B{B}_apply_fwd_ms"] = timed(lambda: L @ x, args.iters)
            r[f"B{B}_apply_fwdbwd_ms"] = timed(lambda: (L @ x).backward(g), args.iters)
            r[f"B{B}_smooth_fwdbwd_ms"] = timed(lambda: uniform_laplacian_smoothing(x, faces).backward(g), args.iters)
            xt = x.detach().permute(1, 0, 2).reshape(V, B * 3)
            r[f"B{B}_torch_csr_mm_ms"] = timed(lambda: torch.sparse.mm(csr, xt) - xt, args.iters)
            # bytes of one L @ x: the CSR (adj_ptr, adj, weight) once and x read ~deg times (cached), y once
            nbytes = 4 * (V + 1 + E + V) + 2 * B * V * 3 * 4
            t = r[f"B{B}_apply_fwd_ms"]
            r[f"B{B}_apply_fwd_MB"] = nbytes / 1e6
            frac = nbytes / (t * 1e-3) / (HBM_GBS * 1e9)
            r[f"B{B}_hbm_fraction"] = frac
            # below half of HBM bandwidth the call is bound by its fixed cost (launch, host-side call), not bytes
            r[f"B{B}_bound"] = "HBM" if frac >= 0.5 else "launch/call latency"
            # check against fp64 on a sample of rows
            y = (L @ x).detach()
            rows = torch.from_numpy(rng.choice(V, min(V, 2048), replace=False)).to(DEV)
            err = 0.0
            ap_, adj, w = topo.adj_ptr.cpu().numpy(), topo.adj.cpu().numpy(), topo.weight.cpu().numpy().astype(np.float64)
            xs = x.detach().cpu().numpy().astype(np.float64)
            yh = y.cpu().numpy()
            for i in rows.cpu().numpy():
                nb = adj[ap_[i]:ap_[i + 1]]
                nb = nb[nb != i]
                err = max(err, float(np.abs(yh[:, i] - (w[i] * xs[:, nb].sum(1) - xs[:, i])).max()))
            r[f"B{B}_rel_err"] = err / float(np.abs(xs).max())
            del x, g, xt
        # the reference's dense path: build once, one matmul per step
        Ld = None
        try:
            r["dense_build_ms"] = timed(lambda: ref_dense_laplacian(V, faces), max(1, args.iters // 4))
            Ld = ref_dense_laplacian(V, faces)
            x1 = torch.randn((1, V, 3), device=DEV)
            r["dense_matmul_B1_ms"] = try_time(lambda: torch.matmul(Ld, x1), args.iters)
        except torch.OutOfMemoryError:
            r["dense_build_ms"] = r["dense_matmul_B1_ms"] = None
        del Ld
        torch.cuda.empty_cache()
        ff = torch.randn((1, F, 3, 3), device=DEV).requires_grad_(True)
        ga = torch.randn((1, V, 3), device=DEV)
        r["average_fwdbwd_ms"] = timed(lambda: mesh.average_face_vertex_features(faces, ff, V).backward(ga), args.iters)
        ffr = ff.detach().clone().requires_grad_(True)
        r["ref_average_fwdbwd_ms"] = timed(lambda: ref_average(faces, ffr, V).backward(ga), args.iters)
        ok = torch.allclose(mesh.average_face_vertex_features(faces, ff.detach(), V), ref_average(faces, ff.detach(), V),
                            rtol=1e-5, atol=1e-6)
        r["average_matches_scatter_add"] = bool(ok)
        results.append(r)
        print(f"level {level}: V {V} F {F} build {r['build_ms']:.3f} ms | "
              f"L@x B1 fwd {r['B1_apply_fwd_ms']:.3f} fwd+bwd {r['B1_apply_fwdbwd_ms']:.3f} ({r['B1_bound']}) | "
              f"B32 fwd {r['B32_apply_fwd_ms']:.3f} fwd+bwd {r['B32_apply_fwdbwd_ms']:.3f} "
              f"({r['B32_bound']}{', %.0f%% of HBM' % (100 * r['B32_hbm_fraction']) if 'B32_hbm_fraction' in r else ''}) | "
              f"smooth B32 fwd+bwd {r['B32_smooth_fwdbwd_ms']:.3f} | torch csr B1 {r['B1_torch_csr_mm_ms']:.3f} "
              f"B32 {r['B32_torch_csr_mm_ms']:.3f} | dense build {fmt(r['dense_build_ms'])} matmul "
              f"{fmt(r['dense_matmul_B1_ms'])} | average fwd+bwd {r['average_fwdbwd_ms']:.3f} vs scatter_add "
              f"{r['ref_average_fwdbwd_ms']:.3f} | rel err {r['B32_rel_err']:.1e}", flush=True)
    print(json.dumps(dict(device=name, power_limit=power, results=results)))


if __name__ == "__main__":
    main()
