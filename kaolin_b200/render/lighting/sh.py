"""Spherical-harmonics diffuse lighting — drop-ins for kaolin.render.lighting.sh (``project_onto_sh9``,
``sh9_irradiance``, ``sh9_diffuse``).  The per-point shading is one sm_90a kernel each way
(kaolin_b200/csrc/lighting.cu, model SH9); ``project_onto_sh9`` of the single light direction is
torch glue in front of it, and autograd carries the coefficients' gradient back to the direction."""
import torch

from ... import _lib
from ..mesh import _host
from .sg import DiffuseB200

__all__ = ["project_onto_sh9", "sh9_irradiance", "sh9_diffuse"]

_Y00 = 0.28209479177            # sqrt(1 / (4 pi))
_Y1 = 0.4886025119              # sqrt(3 / (4 pi))
_Y2 = 1.0925484305920792        # sqrt(15 / (4 pi))
_Y20 = (0.94617469575, 0.31539156525)   # sqrt(5 / (16 pi)) * (3 z^2 - 1)
_Y22 = 0.5462742152960396       # sqrt(15 / (16 pi))


def project_onto_sh9(directions):
    r"""The 9 real spherical-harmonic coefficients (bands 0-2) of cartesian ``directions``: a tensor of
    last dimension 3 (-> last dimension 9) or a list of 3 numbers (-> a (9,) tensor)."""
    if isinstance(directions, torch.Tensor):
        assert directions.shape[-1] == 3
        x, y, z = directions[..., 0], directions[..., 1], directions[..., 2]
        coeffs = [torch.full_like(x, _Y00)]
        stack = lambda cs: torch.stack(cs, dim=-1)
    elif isinstance(directions, list):
        assert len(directions) == 3
        x, y, z = directions
        coeffs = [_Y00]
        stack = torch.tensor
    else:
        raise TypeError(f"directions is a {type(directions)}, must be a list or a torch.Tensor")
    coeffs += [-_Y1 * y, _Y1 * z, -_Y1 * x,
               _Y2 * (x * y), -_Y2 * (y * z), _Y20[0] * (z * z) - _Y20[1], -_Y2 * x * z, _Y22 * (x * x - y * y)]
    return stack(coeffs)


def sh9_irradiance(lights, normals):
    r"""Irradiance (num_points,) at points of normal ``normals`` (num_points, 3) from radiance given by
    9 spherical-harmonic coefficients ``lights`` (9,), the clamped cosine lobe projected on the same
    bands."""
    assert lights.shape == (9,)
    assert normals.ndim == 2 and normals.shape[-1] == 3
    _host.check_tensors("sh9_irradiance", [("lights", lights), ("normals", normals)])
    return DiffuseB200.apply(_lib.LIGHT_SH9, lights, None, None, normals, None)


def sh9_diffuse(directions, normals, albedo):
    r"""Lambertian outgoing radiance (num_points, 3): ``albedo * sh9_irradiance(project_onto_sh9(directions),
    normals)`` for one light direction ``directions`` (3,)."""
    assert directions.shape == (3,)
    assert normals.ndim == 2 and normals.shape[1] == 3
    assert normals.shape == albedo.shape
    _host.check_tensors("sh9_diffuse", [("directions", directions), ("normals", normals), ("albedo", albedo)])
    return DiffuseB200.apply(_lib.LIGHT_SH9, project_onto_sh9(directions), None, None, normals, albedo)
