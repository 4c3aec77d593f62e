"""The general reduced SG inner product at the operator boundary (``kaolin_b200._C.render.sg``) against
the reference's own CUDA operator, at the sizes of the reference's own test (num_sg in {1, 17, 32, 511,
10000} x num_other in {1, 17, 32, 511}), through its stored outputs (tests/golden/ref_cuda_sg.npz,
oracle/ref_golden_sg.py), and against the fp64 restatement (oracle/lighting.py).

The reference's kernels load ``sharpness[sg_idx]`` and ``other_sharpness[other_idx]`` without a bounds
check, up to the next multiple of 32 rows, so they are always given prefix views of buffers padded to a
multiple of 32.  Where the reference's output is further than 1e-5 of scale from fp64, fp64 decides."""
import numpy as np
import pytest
import torch

from oracle import build_ref_sg, ref_golden_sg
from oracle import lighting as OL
from kaolin_b200 import _C as b200_C

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAMES = ("out", "g_a", "g_d", "g_s", "g_oa", "g_od", "g_os")


def _padded(a, rows):
    buf = np.ones((-(-max(rows, 1) // 32) * 32,) + a.shape[1:], np.float32)
    buf[:rows] = a
    return torch.from_numpy(buf).to(DEV)[:rows]


def _inputs(n, m):
    rng = np.random.default_rng(1000 * n + m)
    unit = lambda k: (lambda v: v / np.linalg.norm(v, axis=1, keepdims=True))(rng.normal(size=(k, 3)))
    arrs = [rng.uniform(0, 2, (n, 3)), unit(n), rng.uniform(0.5, 10, n),
            rng.uniform(0, 2, (m, 3)), unit(m), rng.uniform(0.5, 10, m), rng.uniform(-0.3, 0.7, (n, 3))]
    rows = [n, n, n, m, m, m, n]
    return [_padded(a.astype(np.float32), r) for a, r in zip(arrs, rows)]


def _err(a, b, scale):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max()) / max(scale, 1e-30) if a.size else 0.0


@pytest.mark.parametrize("m", [1, 17, 32, 511])
@pytest.mark.parametrize("n", [1, 17, 32, 511, 10000])
def test_general_inner_product_vs_reference_cuda_operator(n, m):
    a, d, s, oa, od, os_, g = _inputs(n, m)

    def live():
        C = build_ref_sg.load()
        assert C is not None, "oracle/_ref/kaolin_ref_sg_C.so is needed to record"
        out = C.unbatched_reduced_sg_inner_product_forward_cuda(a, d, s, oa, od, os_)
        return dict(zip(NAMES, [out] + list(C.unbatched_reduced_sg_inner_product_backward_cuda(g, a, d, s, oa, od, os_))))

    ref = ref_golden_sg.reference(f"sg_{n}x{m}", live, NAMES)
    ours = [b200_C.render.sg.unbatched_reduced_sg_inner_product_forward_cuda(a, d, s, oa, od, os_)]
    ours += b200_C.render.sg.unbatched_reduced_sg_inner_product_backward_cuda(g, a, d, s, oa, od, os_)
    ins64 = [t.double().requires_grad_(True) for t in (a, d, s, oa, od, os_)]
    o64 = OL.reduced_sg_inner_product(*ins64)
    (o64 * g.double()).sum().backward()
    exact = [o64.detach()] + [t.grad for t in ins64]
    for name, mine, e in zip(NAMES, ours, exact):
        scale = float(e.abs().max()) if e.numel() else 0.0
        assert _err(mine.cpu().numpy(), e.cpu().numpy(), scale) <= 1e-5, (name, "vs fp64")
        mine_rows, ref_rows = ref.pair(name, mine)
        e_rows = ref_golden_sg.ref_golden._row_view(name, e.cpu().numpy())[ref.rows(name)]
        ref_err = _err(ref_rows, e_rows, scale)
        if ref_err > 1e-5:
            print(f"[ref_cuda_sg] {n}x{m} {name}: the reference operator is {ref_err:.2e} of scale from fp64")
        else:
            assert _err(mine_rows, ref_rows, scale) <= 1e-5, (name, "vs the reference operator")
