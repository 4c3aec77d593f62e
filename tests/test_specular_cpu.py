"""Specular lighting without a GPU: the fp64 restatement the GPU tests compare against
(oracle/specular.py) and the plain-torch building blocks reproduce the reference's golden vectors
(tests/golden/specular.npz); the public function rejects CPU tensors with the library's wording and
keeps the reference's signature."""
import inspect
import os

import numpy as np
import pytest
import torch

from oracle import ref_import
from oracle import specular as OS
from kaolin_b200.render import lighting

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "specular.npz"))
T = lambda k: torch.from_numpy(np.ascontiguousarray(G[k]))
INPUTS = ("amp", "dir", "sharp", "normal", "roughness", "view", "spec_albedo")


def close(a, ref, tol):
    ref = np.asarray(ref)
    np.testing.assert_allclose(np.asarray(a), ref, rtol=0, atol=tol * max(float(np.abs(ref).max()), 1e-30))


@pytest.mark.parametrize("L", [1, 2, 7, 8, 40])
def test_restatement_matches_the_reference_golden(L):
    ins = [T(f"L{L}_{k}").requires_grad_(True) for k in INPUTS]
    o = OS.sg_warp_specular_term(*ins)
    close(o.detach(), G[f"L{L}_out"], 1e-12)
    (o * T(f"L{L}_w")).sum().backward()
    for k, t in zip(INPUTS, ins):
        close(t.grad, G[f"L{L}_g_{k}"], 1e-12)


def test_building_blocks_match_the_reference_golden():
    amp, d, s = lighting.sg_distribution_term(T("bb_normal"), T("bb_roughness"))
    assert amp.shape == (G["bb_normal"].shape[0], 3)
    close(amp, G["bb_ndf_amp"], 1e-15); close(d, G["bb_ndf_dir"], 0); close(s, G["bb_ndf_sharp"], 1e-15)
    wa, wd, ws = lighting.sg_warp_distribution(amp, d, s, T("bb_view"))
    close(wa, G["bb_warp_amp"], 0); close(wd, G["bb_warp_dir"], 1e-15); close(ws, G["bb_warp_sharp"], 1e-15)
    close(lighting.fresnel(T("bb_ldh"), T("bb_spec_albedo")), G["bb_fresnel"], 1e-15)
    # the restatement's lobe is the two building blocks composed
    la, lw, ls = OS.lobe(T("bb_normal"), T("bb_roughness"), T("bb_view"))
    close(la, G["bb_warp_amp"], 1e-15); close(lw, G["bb_warp_dir"], 1e-15); close(ls, G["bb_warp_sharp"], 1e-15)


def test_cpu_inputs_are_rejected():
    args = (torch.rand(2, 3), torch.rand(2, 3), torch.rand(2), torch.rand(5, 3), torch.rand(5) + 0.3,
            torch.rand(5, 3), torch.rand(5, 3))
    with pytest.raises(RuntimeError, match="expected .* to be a CUDA tensor \\(kaolin_b200 has no CPU path\\)"):
        lighting.sg_warp_specular_term(*args)


@pytest.mark.skipif(not ref_import.available(), reason="the reference's Python sources are not present")
def test_signatures_match_the_reference():
    sg = ref_import.module("kaolin.render.lighting.sg")
    for name in ("sg_warp_specular_term", "sg_distribution_term", "sg_warp_distribution", "fresnel"):
        ref = getattr(sg, name)
        ref_params = list(inspect.signature(ref).parameters) if not hasattr(ref, "schema") else \
            [a.name for a in ref.schema.arguments]
        assert list(inspect.signature(getattr(lighting, name)).parameters) == ref_params, name
