"""kaolin.ops.conversions drop-ins on sm_90a kernels: marching tetrahedra, marching cubes and
voxelization of meshes and point clouds."""
from .pointcloud import pointclouds_to_voxelgrids  # noqa: F401
from .tetmesh import MarchingTetrahedra, marching_tetrahedra  # noqa: F401
from .trianglemesh import trianglemeshes_to_voxelgrids  # noqa: F401
from .voxelgrid import unbatched_mcube_forward, voxelgrids_to_trianglemeshes  # noqa: F401

__all__ = ["marching_tetrahedra", "MarchingTetrahedra", "voxelgrids_to_trianglemeshes", "unbatched_mcube_forward",
           "trianglemeshes_to_voxelgrids", "pointclouds_to_voxelgrids"]
