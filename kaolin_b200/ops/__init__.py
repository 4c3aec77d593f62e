"""kaolin.ops drop-ins: the mesh Laplacian, adjacency, vertex averaging, Loop subdivision, tet-mesh
subdivision, marching tetrahedra, marching cubes (``voxelgrids_to_trianglemeshes``), cubic meshes
(``voxelgrids_to_cubic_meshes``) and the point-in-mesh test (``check_sign``), surface sampling
(``sample_points``, ``face_areas``) and the voxel-grid operators
(``voxelgrid.fill``, ``extract_surface``, ``extract_odms``, ``project_odms``) and farthest point sampling
(``pointcloud.farthest_point_sampling``, with ``pointcloud.center_points``) on sm_90a kernels."""
from . import mesh  # noqa: F401
from . import conversions  # noqa: F401
from . import voxelgrid  # noqa: F401
from . import pointcloud  # noqa: F401
