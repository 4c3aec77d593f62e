"""The specular kernel (sg_warp_specular_term, kaolin_b200/csrc/lighting.cu) against two torch paths
on one GPU: N = 2^24 shaded points, L lights.

    python scripts/bench_specular.py [--n 16777216] [--lights 1,2,8,32,128] [--min-seconds 0.5]

For every L: CUDA-event times of the forward, of forward+backward with all gradients and of
forward+backward with light gradients only, for
  * "ours":     the fused kernels;
  * "torch":    the reference formulation in fp32 torch (oracle/specular.py over oracle/lighting.py,
                with its (N, L, 3) temporaries);
  * "composed": the reference's structure with the torch prologue and epilogue around this library's
                general SG inner product (kaolin_b200.render.lighting.unbatched_reduced_sg_inner_product);
  * "ref op":   the same structure around the reference's own CUDA operator (oracle/_ref, built by
                oracle/build_ref_sg.py) at L >= 8, where the reference uses it, when it is built.
The kernels' output and every gradient are checked against the fp64 restatement on well-conditioned
inputs (unit view, unit normal with n.v in [0.2, 1], roughness in [0.3, 1]) over all N points, in
chunks, next to the error of the reference formulation evaluated in fp32 on the same inputs.  The
script fails where an error exceeds both 1e-5 of scale and 4x the fp32 formulation's: the roughness
gradient is a near cancellation of the lobe's amplitude and sharpness terms, and over 2^24 points
fp32 torch itself can exceed 1e-5 there.  It reports the binding limit (HBM bytes at 3.35 TB/s,
or FP32 / SFU issue at the SM clock) and the fraction of it reached, and prints the device name and
power limit, then one JSON line.
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
from oracle import specular as OS  # noqa: E402
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


def cost(N, L, phase, point_grads):
    """(bytes, fp32 ops, sfu ops) the algorithm needs.  Forward: normal, roughness, view, spec_albedo
    read, out written (52 B/point).  Backward: the same inputs and grad_out read (52 B/point), plus
    grad_normal, grad_roughness, grad_view and grad_spec_albedo written (40 B/point) when per-point
    gradients are requested: 92 B/point.  Per (point, light) pair the SG inner product of the general
    op: 20 fp32 ops and 4 SFU ops forward, three times that backward (recompute + gradient)."""
    byt = 52 * N + (40 * N if phase == "bwd" and point_grads else 0)
    mult = 1 if phase == "fwd" else 3
    return byt, N * L * 20 * mult, N * L * 4 * mult


def _pad32(t):
    """Prefix view of a buffer padded to a multiple of 32 rows: the reference's kernels load sharpness
    up to the next multiple of 32 rows without a bounds check."""
    rows = t.shape[0]
    buf = torch.ones((-(-rows // 32) * 32,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    buf[:rows] = t
    return buf[:rows]


def ref_operator_inner(C):
    """unbatched_reduced_sg_inner_product through the reference's own CUDA operator."""
    class RefOp(torch.autograd.Function):
        @staticmethod
        def forward(ctx, *ins):
            ins = [_pad32(t.contiguous()) for t in ins]
            ctx.save_for_backward(*ins)
            return C.unbatched_reduced_sg_inner_product_forward_cuda(*ins)

        @staticmethod
        def backward(ctx, g):
            return tuple(C.unbatched_reduced_sg_inner_product_backward_cuda(g.contiguous(), *ctx.saved_tensors))
    return RefOp.apply


def points(N, gen, dev):
    v = torch.nn.functional.normalize(torch.randn((N, 3), device=dev, generator=gen), dim=-1)
    t = torch.randn((N, 3), device=dev, generator=gen)
    t = torch.nn.functional.normalize(t - (t * v).sum(1, keepdim=True) * v, dim=-1)
    c = 0.2 + 0.8 * torch.rand((N, 1), device=dev, generator=gen)
    n = c * v + torch.sqrt(1 - c * c) * t
    del t
    r = 0.3 + 0.7 * torch.rand((N,), device=dev, generator=gen)
    return [n, r, v, torch.rand((N, 3), device=dev, generator=gen)]


def check(lights, pts, g, chunk=1 << 17):
    """Max error of the kernels' output and gradients ("err_*") and of the reference formulation in
    fp32 ("torch32_err_*") relative to the scale of the fp64 restatement, over all N points (both torch
    paths evaluated chunk by chunk; their light gradients summed over chunks)."""
    lp = [t.clone().requires_grad_(True) for t in lights]
    pp = [t.clone().requires_grad_(True) for t in pts]
    o = lighting.sg_warp_specular_term(*lp, *pp)
    (o * g).sum().backward()
    names = ("out", "g_normal", "g_roughness", "g_view", "g_spec_albedo")
    mine = dict(zip(names, [o.detach()] + [t.grad for t in pp]))
    l64 = [t.double().requires_grad_(True) for t in lights]
    l32 = [t.clone().requires_grad_(True) for t in lights]
    err, err32, scale = {}, {}, {}

    def upd(k, a, a32, b):
        err[k] = max(err.get(k, 0.), float((a.double() - b).abs().max()))
        err32[k] = max(err32.get(k, 0.), float((a32.double() - b).abs().max()))
        scale[k] = max(scale.get(k, 0.), float(b.abs().max()))
    for i in range(0, pts[0].shape[0], chunk):
        sl = slice(i, i + chunk)
        p64 = [t[sl].double().requires_grad_(True) for t in pts]
        r = OS.sg_warp_specular_term(*l64, *p64)
        (r * g[sl].double()).sum().backward()
        p32 = [t[sl].clone().requires_grad_(True) for t in pts]
        r32 = OS.sg_warp_specular_term(*l32, *p32)
        (r32 * g[sl]).sum().backward()
        for k, ref, ref32 in zip(names, [r.detach()] + [t.grad for t in p64], [r32.detach()] + [t.grad for t in p32]):
            upd(k, mine[k][sl], ref32, ref)
    for k, a, a32, b in zip(("g_amp", "g_dir", "g_sharp"), lp, l32, l64):
        upd(k, a.grad, a32.grad, b.grad)
    return ({f"err_{k}": err[k] / max(scale[k], 1e-30) for k in err},
            {f"torch32_err_{k}": err32[k] / max(scale[k], 1e-30) for k in err})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 24)
    ap.add_argument("--lights", default="1,2,8,32,128")
    ap.add_argument("--min-seconds", type=float, default=0.5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_specular.py measures on a CUDA device"
    dev = torch.device("cuda")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"device: {torch.cuda.get_device_name(0)}; nvidia-smi: {q}")
    gen = torch.Generator(device=dev); gen.manual_seed(0)
    N = args.n
    pts = points(N, gen, dev)
    g = torch.rand((N, 3), device=dev, generator=gen)
    ref_op = build_ref_sg.load()
    print("reference CUDA operator:", "oracle/_ref/kaolin_ref_sg_C.so" if ref_op is not None else "not built (not measured)")
    paths = {"ours": lighting.sg_warp_specular_term,
             "torch": OS.sg_warp_specular_term,
             "composed": lambda *a: OS.sg_warp_specular_term(*a, inner=lighting.unbatched_reduced_sg_inner_product)}
    if ref_op is not None:
        ref_inner = ref_operator_inner(ref_op)
        paths["refop"] = lambda *a: OS.sg_warp_specular_term(*a, inner=ref_inner)
    rows = []
    for L in [int(x) for x in args.lights.split(",")]:
        amp = torch.rand((L, 3), device=dev, generator=gen) * 2
        d = torch.nn.functional.normalize(torch.randn((L, 3), device=dev, generator=gen), dim=-1)
        s = torch.exp(torch.rand((L,), device=dev, generator=gen) * math.log(100.)) * 0.5
        row = {"L": L, "N": N}
        for impl, fn in paths.items():
            if impl == "refop" and L < 8:
                continue
            lp = [t.clone().requires_grad_(True) for t in (amp, d, s)]
            pp = [t.clone().requires_grad_(True) for t in pts]
            try:
                with torch.no_grad():
                    row[f"{impl}_fwd_ms"] = timed(lambda: fn(*lp, *pts), args.min_seconds)
                row[f"{impl}_fwdbwd_all_ms"] = timed(lambda: (fn(*lp, *pp) * g).sum().backward(), args.min_seconds)
                row[f"{impl}_fwdbwd_lights_ms"] = timed(lambda: (fn(*lp, *pts) * g).sum().backward(), args.min_seconds)
            except torch.OutOfMemoryError:
                row[f"{impl}_fwd_ms"] = "out of memory"
            del lp, pp
            torch.cuda.empty_cache()
        errs, errs32 = check((amp, d, s), pts, g)
        row.update(errs)
        row.update(errs32)
        bad = {k: v for k, v in errs.items() if v > max(1e-5, 4 * errs32["torch32_" + k])}
        assert not bad, (L, bad)
        for phase, key, pg in (("fwd", "ours_fwd_ms", False), ("bwd", "ours_fwdbwd_all_ms", True),
                               ("bwd", "ours_fwdbwd_lights_ms", False)):
            byt, fl, sfu = cost(N, L, phase, pg)
            if phase == "bwd":
                b2, f2, s2 = cost(N, L, "fwd", False)
                byt, fl, sfu = byt + b2, fl + f2, sfu + s2
            bound = max(("HBM", byt / HBM), ("FP32", fl / FP32_OPS), ("SFU", sfu / SFU_OPS), key=lambda x: x[1])
            row[key.replace("_ms", "_bound")] = bound[0]
            row[key.replace("_ms", "_frac")] = round(bound[1] * 1e3 / row[key], 3)
        rows.append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"bench": "specular", "device": torch.cuda.get_device_name(0), "nvidia_smi": q, "rows": rows}))


if __name__ == "__main__":
    main()
