"""Diffuse lighting without a GPU: the ``kaolin_b200._C.render.sg`` shims take the arity of the
reference's call sites and are reached by the reference's own sg.py; the public functions reject
CPU tensors with the library's wording (float64 and non-contiguous inputs need a GPU:
tests/test_lighting_gpu.py); the
fp64 restatement the GPU tests compare against (oracle/lighting.py) reproduces the reference's golden
outputs."""
import inspect
import os

import numpy as np
import pytest
import torch

from oracle import lighting as OL
from oracle import ref_import
from kaolin_b200 import _C as b200_C
from kaolin_b200.render import lighting

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "lighting.npz"))
T = lambda k: torch.from_numpy(np.ascontiguousarray(G[k]))


def test_sg_shims_take_the_arity_of_the_reference_call_sites():
    sig = lambda f: len(inspect.signature(f).parameters)
    assert sig(b200_C.render.sg.unbatched_reduced_sg_inner_product_forward_cuda) == 6    # sg.py:624-626
    assert sig(b200_C.render.sg.unbatched_reduced_sg_inner_product_backward_cuda) == 7   # sg.py:635-637


@pytest.mark.skipif(not ref_import.available(), reason="the reference's Python sources are not present")
def test_reference_sg_module_reaches_the_shims():
    ref_import.setup(b200_C)
    sg = ref_import.module("kaolin.render.lighting.sg")
    sg._C = b200_C
    a, d, s = torch.rand(4, 3), torch.rand(4, 3), torch.rand(4)
    oa, od, os_ = torch.rand(9, 3), torch.rand(9, 3), torch.rand(9)     # >= 8 lobes: the operator path
    with pytest.raises(RuntimeError, match="no CPU path"):
        sg.unbatched_reduced_sg_inner_product(a, d, s, oa, od, os_)
    with pytest.raises(RuntimeError, match="no CPU path"):
        sg.sg_diffuse_inner_product(oa, od, os_, torch.rand(4, 3), torch.rand(4, 3))


@pytest.mark.parametrize("fn,args", [
    (lighting.sg_diffuse_inner_product, lambda: (torch.rand(2, 3), torch.rand(2, 3), torch.rand(2), torch.rand(5, 3), torch.rand(5, 3))),
    (lighting.sg_diffuse_fitted, lambda: (torch.rand(2, 3), torch.rand(2, 3), torch.rand(2), torch.rand(5, 3), torch.rand(5, 3))),
    (lighting.sg_irradiance_inner_product, lambda: (torch.rand(2, 3), torch.rand(2, 3), torch.rand(2), torch.rand(5, 3))),
    (lighting.sh9_irradiance, lambda: (torch.rand(9), torch.rand(5, 3))),
    (lighting.sh9_diffuse, lambda: (torch.rand(3), torch.rand(5, 3), torch.rand(5, 3))),
    (lighting.unbatched_reduced_sg_inner_product, lambda: (torch.rand(4, 3), torch.rand(4, 3), torch.rand(4),
                                                           torch.rand(2, 3), torch.rand(2, 3), torch.rand(2))),
])
def test_cpu_and_float64_inputs_are_rejected(fn, args):
    with pytest.raises(RuntimeError, match="expected .* to be a CUDA tensor \\(kaolin_b200 has no CPU path\\)"):
        fn(*args())


def test_operator_shim_error_wording():
    f = b200_C.render.sg.unbatched_reduced_sg_inner_product_forward_cuda
    args = [torch.rand(4, 3), torch.rand(4, 3), torch.rand(4), torch.rand(2, 3), torch.rand(2, 3), torch.rand(2)]
    with pytest.raises(RuntimeError, match="no CPU path"):
        f(*args)


@pytest.mark.parametrize("L", [1, 2, 7, 8, 40])
def test_restatement_matches_the_reference_golden(L):
    amp, d, s, n, al = (T(f"L{L}_{k}") for k in ("amp", "dir", "sharp", "normal", "albedo"))
    np.testing.assert_allclose(OL.sg_irradiance_inner_product(amp, d, s, n).numpy(), G[f"L{L}_irr_ip_out"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(OL.sg_diffuse_inner_product(amp, d, s, n, al).numpy(), G[f"L{L}_diff_ip_out"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(OL.sg_diffuse_fitted(amp, d, s, n, al).numpy(), G[f"L{L}_fitted_out"], rtol=1e-12, atol=1e-12)


def test_restatement_matches_the_reference_golden_sh9():
    np.testing.assert_allclose(OL.sh9_diffuse(T("sh_direction"), T("sh_normal"), T("sh_albedo")).numpy(),
                               G["sh_diffuse_out"], rtol=1e-9, atol=1e-10)
    np.testing.assert_allclose(OL.sh9_irradiance(T("sh_lights"), T("sh_normal")).numpy(), G["sh_irr_out"], rtol=1e-9, atol=1e-10)
    np.testing.assert_allclose(lighting.project_onto_sh9(T("sh_direction")).numpy(), G["sh_project"], rtol=1e-12)
    np.testing.assert_allclose(lighting.project_onto_sh9([float(v) for v in G["sh_direction"]]).numpy(),
                               G["sh_project"].astype(np.float32), rtol=1e-6)
