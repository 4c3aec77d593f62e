"""Diffuse-lighting kernels (kaolin_b200/csrc/lighting.cu) against the reference formulation in torch
(oracle/lighting.py, fp32) on one GPU: N = 2^24 shaded points, L lights, three models.

    python scripts/bench_lighting.py [--n 16777216] [--lights 1,2,8,32,128] [--min-seconds 0.5]

For every (model, L): CUDA-event times of the forward and of forward+backward with all gradients and
with light gradients only, for both, and for the SG inner product also the reference's own CUDA
operator (oracle/_ref, built by oracle/build_ref_sg.py) when present, given inputs padded to a multiple
of 32 rows; the bound that applies (HBM bytes at 3.35 TB/s or FP32/SFU issue at the SM clock) and the
fraction of it reached.  The kernels' outputs and every gradient are checked against the fp64
restatement at the timed size (in chunks of points); the script fails above 1e-5 of scale.  For the
fitted model the normal gradient skips points at its two clamp kinks (mu = 1, mean = 0) that fp32
rounding may cross (oracle/lighting.fitted_kinks).  Prints the device name and power limit, then one JSON line.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
from oracle import build_ref_sg  # noqa: E402
from oracle import lighting as OL  # noqa: E402
from kaolin_b200.render import lighting  # noqa: E402

HBM = 3.35e12
# FP32 issue: 132 SMs x 128 lanes x 2 (FMA) at the boost clock; MUFU (ex2, rsqrt, rcp): 16/SM/clk
SMS, CLK = 132, 1.98e9
FP32_OPS, SFU_OPS = SMS * 128 * CLK, SMS * 16 * CLK


def timed(fn, min_s):
    fn(); torch.cuda.synchronize()
    t0 = time.perf_counter(); fn(); torch.cuda.synchronize()
    reps = max(3, int(min_s / max(time.perf_counter() - t0, 1e-6)))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def cost(model, N, L, phase, point_grads):
    """(bytes, fp32 ops, sfu ops) the algorithm needs.  Forward: normal + albedo read, out written
    (36 B/point).  Backward: grad_out + normal + albedo read (36 B/point), plus grad_normal + grad_albedo
    written (24 B/point) when per-point gradients are requested."""
    if phase == "fwd":
        byt = 36 * N
    else:
        byt = 36 * N + (24 * N if point_grads else 0)
    pairs = N * (1 if model == "sh9" else L)
    per = {"ip": (20, 4), "fitted": (12, 0), "sh9": (25, 0)}[model]      # fp32 ops, SFU ops per pair (forward)
    mult = 1 if phase == "fwd" else 3                                        # backward: recompute + gradient
    return byt, pairs * per[0] * mult, pairs * per[1] * mult


def _pad32(t):
    """Prefix view of a buffer padded to a multiple of 32 rows: the reference's kernels load sharpness
    up to the next multiple of 32 rows without a bounds check."""
    rows = t.shape[0]
    buf = torch.ones((-(-rows // 32) * 32,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    buf[:rows] = t
    return buf[:rows]


def time_reference_operator(C, lights, n, al, g, min_s):
    """sg_diffuse_inner_product at the reference's operator boundary: the cosine lobe, the operator,
    clamp and albedo / pi (sg.py:514-558); the backward runs the operator's backward."""
    N = n.shape[0]
    la, ls = _pad32(torch.full_like(n, 1.17)), _pad32(torch.full((N,), 2.133, device=n.device))
    nn = _pad32(n)
    oa, od, os_ = (_pad32(t) for t in lights)

    def fwd():
        return torch.clamp(C.unbatched_reduced_sg_inner_product_forward_cuda(la, nn, ls, oa, od, os_), min=0.) * (al / math.pi)

    def fwdbwd():
        pre = C.unbatched_reduced_sg_inner_product_forward_cuda(la, nn, ls, oa, od, os_)
        gpre = torch.where(pre >= 0, g * (al / math.pi), torch.zeros_like(g)).contiguous()
        C.unbatched_reduced_sg_inner_product_backward_cuda(gpre, la, nn, ls, oa, od, os_)

    return {"ref_cuda_fwd_ms": timed(fwd, min_s), "ref_cuda_fwdbwd_all_ms": timed(fwdbwd, min_s)}


def check(model, ours, ref, lights, n, al, g, chunk=1 << 17):
    """Max error of the kernels' output and gradients relative to the scale of the fp64 restatement,
    over all N points (fp64 evaluated chunk by chunk; the light gradients summed over chunks)."""
    lp = [t.clone().requires_grad_(True) for t in lights]
    pp = [n.clone().requires_grad_(True), al.clone().requires_grad_(True)]
    o = ours(*lp, *pp)
    (o * g).sum().backward()
    mine = {"out": o.detach(), "g_normal": pp[0].grad, "g_albedo": pp[1].grad}
    l64 = [t.double().requires_grad_(True) for t in lights]
    err, scale = {}, {}
    upd = lambda k, a, b: (err.__setitem__(k, max(err.get(k, 0.), float((a.double() - b).abs().max()))),
                           scale.__setitem__(k, max(scale.get(k, 0.), float(b.abs().max()))))
    for i in range(0, n.shape[0], chunk):
        sl = slice(i, i + chunk)
        p64 = [n[sl].double().requires_grad_(True), al[sl].double().requires_grad_(True)]
        r = ref(*l64, *p64)
        (r * g[sl].double()).sum().backward()
        keep = slice(None)
        if model == "fitted":      # compare away from the clamp kinks that fp32 rounding may cross
            kink, rounding_only = OL.fitted_kinks(*[t.detach() for t in l64], p64[0].detach(), mine["g_albedo"][sl], g[sl])
            assert rounding_only, "a clamp flip not explained by fp32 rounding"
            keep = ~kink
        upd("out", mine["out"][sl], r.detach()); upd("g_normal", mine["g_normal"][sl][keep], p64[0].grad[keep])
        upd("g_albedo", mine["g_albedo"][sl], p64[1].grad)
    for k, a, b in zip(("g_amp", "g_dir", "g_sharp"), lp, l64):
        if b.grad is not None:
            upd(k, a.grad, b.grad)
    return {f"err_{k}": err[k] / max(scale[k], 1e-30) for k in err}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 24)
    ap.add_argument("--lights", default="1,2,8,32,128")
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--no-torch", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_lighting.py measures on a CUDA device"
    dev = torch.device("cuda")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"device: {torch.cuda.get_device_name(0)}; nvidia-smi: {q}")
    gen = torch.Generator(device=dev); gen.manual_seed(0)
    N = args.n
    n = torch.nn.functional.normalize(torch.randn((N, 3), device=dev, generator=gen), dim=-1)
    al = torch.rand((N, 3), device=dev, generator=gen)
    g = torch.rand((N, 3), device=dev, generator=gen)
    ref_op = build_ref_sg.load()
    print("reference CUDA operator:", "oracle/_ref/kaolin_ref_sg_C.so" if ref_op is not None else "not built (not measured)")
    rows = []
    for L in [int(x) for x in args.lights.split(",")]:
        amp = torch.rand((L, 3), device=dev, generator=gen) * 2
        d = torch.nn.functional.normalize(torch.randn((L, 3), device=dev, generator=gen), dim=-1)
        s = torch.exp(torch.rand((L,), device=dev, generator=gen) * math.log(100.)) * 0.5
        for model, ours, ref in (("ip", lighting.sg_diffuse_inner_product, OL.sg_diffuse_inner_product),
                                 ("fitted", lighting.sg_diffuse_fitted, OL.sg_diffuse_fitted),
                                 ("sh9", lambda a, dd, ss, nn, aa: lighting.sh9_diffuse(dd[0], nn, aa),
                                  lambda a, dd, ss, nn, aa: OL.sh9_diffuse(dd[0], nn, aa))):
            if model == "sh9" and L != 1:
                continue
            row = {"model": model, "L": L, "N": N}
            for impl, fn in (("ours", ours), ("torch", ref)):
                if impl == "torch" and args.no_torch:
                    continue
                lp = [t.clone().requires_grad_(True) for t in (amp, d, s)]
                pp = [n.clone().requires_grad_(True), al.clone().requires_grad_(True)]
                pl = [n, al]
                try:
                    with torch.no_grad():
                        row[f"{impl}_fwd_ms"] = timed(lambda: fn(*lp, *pl), args.min_seconds)
                    row[f"{impl}_fwdbwd_all_ms"] = timed(lambda: (fn(*lp, *pp) * g).sum().backward(), args.min_seconds)
                    row[f"{impl}_fwdbwd_lights_ms"] = timed(lambda: (fn(*lp, *pl) * g).sum().backward(), args.min_seconds)
                except torch.OutOfMemoryError:
                    row[f"{impl}_fwd_ms"] = "out of memory"
                torch.cuda.empty_cache()
            if model == "ip" and ref_op is not None:
                row.update(time_reference_operator(ref_op, (amp, d, s), n, al, g, args.min_seconds))
            errs = check(model, ours, ref, (amp, d, s), n, al, g)
            row.update(errs)
            bad = {k: v for k, v in errs.items() if v > 1e-5}
            assert not bad, (model, L, bad)
            for phase, key, pg in (("fwd", "ours_fwd_ms", False), ("bwd", "ours_fwdbwd_all_ms", True),
                                   ("bwd", "ours_fwdbwd_lights_ms", False)):
                byt, fl, sfu = cost(model, N, L, phase, pg)
                if phase == "bwd":
                    b2, f2, s2 = cost(model, N, L, "fwd", False)
                    byt, fl, sfu = byt + b2, fl + f2, sfu + s2
                t_hbm, t_fp, t_sfu = byt / HBM, fl / FP32_OPS, sfu / SFU_OPS
                bound = max(("HBM", t_hbm), ("FP32", t_fp), ("SFU", t_sfu), key=lambda x: x[1])
                row[key.replace("_ms", "_bound")] = bound[0]
                row[key.replace("_ms", "_frac")] = round(bound[1] * 1e3 / row[key], 3)
            rows.append(row)
            print(json.dumps(row), flush=True)
    print(json.dumps({"bench": "lighting", "device": torch.cuda.get_device_name(0), "nvidia_smi": q, "rows": rows}))


if __name__ == "__main__":
    main()
