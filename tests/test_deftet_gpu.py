"""DefTet volumetric renderer on sm_90a (kaolin_b200/csrc/deftet.cu; SURVEY.md §8f rank 3) against the
golden vectors of the reference's own pure-PyTorch oracle (tests/golden/deftet.npz) and the numpy /
torch restatements in oracle/deftet.py — including what the small scenes do not reach: truncation at
knum (first knum faces BY INDEX, deftet_cuda.cu:155-171), faces wider than the binning grid allows
(the per-view wide list) and points with more hits than the in-kernel buffer (ordered fallback scan)."""
import os

import numpy as np
import pytest
import torch

from oracle import deftet as DT
from kaolin_b200 import _C as b200_C
from kaolin_b200 import _lib
from kaolin_b200.render.mesh import deftet_sparse_render

pytestmark = pytest.mark.gpu
DEV = "cuda"
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "deftet.npz"))


def T(a, grad=False):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV).requires_grad_(grad)


def close(a, ref, tol):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    ref = ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else ref
    err = float(np.abs(a - ref).max()) / max(float(np.abs(ref).max()), 1e-30)
    assert err <= tol, err


@pytest.mark.parametrize("tag", ["soup", "layers"])
def test_deftet_vs_reference_naive_golden(tag):
    knum = int(G[f"{tag}_knum"])
    fvi, ff = T(G[f"{tag}_fvi"], True), T(G[f"{tag}_ff"], True)
    feat, idx = deftet_sparse_render(T(G[f"{tag}_pix"]), T(G[f"{tag}_rr"]), T(G[f"{tag}_fvz"]), fvi, ff, knum)
    assert np.array_equal(idx.cpu().numpy(), G[f"{tag}_idx"])
    close(feat, G[f"{tag}_feat"], 1e-5)
    (feat * T(G[f"{tag}_gw"])).sum().backward()
    close(ff.grad, G[f"{tag}_g_ff"], 1e-5)
    close(fvi.grad, G[f"{tag}_g_fvi"], 1e-4)     # k3^2 in the denominator; the reference's own tests use 1e-3..1e-2


def _scene(B, F, P, spread, size, seed):
    g = torch.Generator().manual_seed(seed)
    c = (torch.rand((B, F, 1, 2), generator=g) * 2 - 1) * spread
    fvi = c + (torch.rand((B, F, 3, 2), generator=g) - 0.5) * size
    fvz = -(torch.rand((B, F, 3), generator=g) * 3 + 1)
    ff = torch.rand((B, F, 3, 3), generator=g)
    pix = (torch.rand((B, P, 2), generator=g) * 2 - 1) * spread
    rr = torch.stack([torch.full((B, P), -3.6), torch.full((B, P), -1.1)], -1)
    return fvi.numpy(), fvz.numpy(), ff.numpy(), pix.numpy(), rr.numpy()


@pytest.mark.parametrize("name,args,knum", [
    ("mesh_like_20k_faces", (2, 20000, 3000, 0.95, 0.03, 1), 30),          # small faces: the grid does the work
    ("truncation_first_knum_by_index", (1, 400, 500, 0.4, 0.8, 2), 6),     # ~40 hits per point, knum 6
    ("wide_faces", (2, 600, 800, 0.9, 1.5, 3), 300),                       # every face spans > 16 cells: wide list
    ("more_hits_than_the_buffer", (1, 900, 60, 0.05, 1.8, 4), 300),        # > 128 hits per point: ordered fallback
])
def test_deftet_operator_vs_oracle(name, args, knum):
    fvi, fvz, ff, pix, rr = _scene(*args)
    bb = np.concatenate([fvi.min(2), fvi.max(2)], -1)
    o_idx, o_d, o_w0, o_w1 = DT.forward_op(fvz, fvi, bb, pix, rr, knum, 1e-8)
    idx, d, w0, w1 = b200_C.render.mesh.deftet_sparse_render_forward_cuda(T(fvz), T(fvi), T(bb), T(pix), T(rr), knum, 1e-8)
    hits = (o_idx >= 0).sum(-1)
    print(f"\n[{name}] hits per point mean {hits.mean():.1f} max {hits.max()}")
    if name == "more_hits_than_the_buffer":
        assert hits.max() > 128
    if name == "truncation_first_knum_by_index":
        assert (hits == knum).mean() > 0.5
    assert np.array_equal(idx.cpu().numpy(), o_idx)                       # same faces, same (index) order
    m = o_idx >= 0
    np.testing.assert_allclose(d.cpu().numpy()[m], o_d[m], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(w0.cpu().numpy()[m], o_w0[m], rtol=0, atol=2e-5)
    np.testing.assert_allclose(w1.cpu().numpy()[m], o_w1[m], rtol=0, atol=2e-5)
    assert np.all(np.isneginf(d.cpu().numpy()[~m])) and np.all(w0.cpu().numpy()[~m] == 0)


def test_deftet_public_api_and_gradients_vs_torch_restatement():
    fvi, fvz, ff, pix, rr = _scene(2, 1500, 700, 0.8, 0.25, 9)
    knum = 24
    t_fvi, t_ff = T(fvi, True), T(ff, True)
    (fa, fb), idx = deftet_sparse_render(T(pix), T(rr), T(fvz), t_fvi, [t_ff[..., :1], t_ff[..., 1:]], knum)
    assert fa.shape[-1] == 1 and fb.shape[-1] == 2 and idx.dtype == torch.int64
    feat = torch.cat([fa, fb], -1)
    r_fvi, r_ff = T(fvi, True), T(ff, True)
    r_feat, r_idx = DT.sparse_render_torch(T(pix), T(rr), T(fvz), r_fvi, r_ff, knum)
    assert torch.equal(idx, r_idx)
    close(feat, r_feat, 1e-5)
    gen = torch.Generator(device=DEV); gen.manual_seed(5)
    gw = torch.rand(feat.shape, device=DEV, generator=gen)
    (feat * gw).sum().backward(); (r_feat * gw).sum().backward()
    close(t_ff.grad, r_ff.grad, 1e-5)
    close(t_fvi.grad, r_fvi.grad, 1e-4)


def test_workspace_at_an_odd_address(monkeypatch):
    """Every workspace starting at byte 1 of a larger buffer: the outputs of an aligned one."""
    fvi, fvz, ff, pix, rr = _scene(2, 1500, 700, 0.8, 0.25, 9)
    bb = np.concatenate([fvi.min(2), fvi.max(2)], -1)

    def run():
        return b200_C.render.mesh.deftet_sparse_render_forward_cuda(T(fvz), T(fvi), T(bb), T(pix), T(rr), 24, 1e-8)

    want = run()
    scratch, odd = _lib.scratch, []
    monkeypatch.setattr(_lib, "scratch", lambda n, device: odd.append(n) or scratch(int(n) + 1, device)[1:])
    got = run()
    assert odd
    for a, b in zip(want, got):
        assert torch.equal(a, b)
