"""kaolin.ops.conversions drop-ins on sm_90a kernels: marching tetrahedra, marching cubes, cubic meshes
from voxel grids and voxelization of meshes and point clouds."""
from .pointcloud import pointclouds_to_voxelgrids  # noqa: F401
from .tetmesh import MarchingTetrahedra, marching_tetrahedra  # noqa: F401
from .trianglemesh import trianglemeshes_to_voxelgrids  # noqa: F401
from .voxelgrid import unbatched_mcube_forward, voxelgrids_to_cubic_meshes, voxelgrids_to_trianglemeshes  # noqa: F401

__all__ = ["marching_tetrahedra", "MarchingTetrahedra", "voxelgrids_to_trianglemeshes", "voxelgrids_to_cubic_meshes",
           "unbatched_mcube_forward", "trianglemeshes_to_voxelgrids", "pointclouds_to_voxelgrids"]
