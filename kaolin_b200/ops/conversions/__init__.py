"""kaolin.ops.conversions drop-ins on sm_90a kernels: marching tetrahedra."""
from .tetmesh import MarchingTetrahedra, marching_tetrahedra  # noqa: F401

__all__ = ["marching_tetrahedra", "MarchingTetrahedra"]
