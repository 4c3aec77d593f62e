"""kaolin.ops.conversions drop-ins on sm_90a kernels: marching tetrahedra and marching cubes."""
from .tetmesh import MarchingTetrahedra, marching_tetrahedra  # noqa: F401
from .voxelgrid import unbatched_mcube_forward, voxelgrids_to_trianglemeshes  # noqa: F401

__all__ = ["marching_tetrahedra", "MarchingTetrahedra", "voxelgrids_to_trianglemeshes", "unbatched_mcube_forward"]
