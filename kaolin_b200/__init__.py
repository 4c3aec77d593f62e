"""kaolin_b200 — H100-native (sm_90a) drop-in for Kaolin's DIB-R hot path.

Provided: ``kaolin.render.mesh.{rasterize, dibr_soft_mask, dibr_rasterization}``
(forward + backward), the four ``kaolin._C.render.mesh.*`` operators, and the steps
either side of the rasterizer in the DIB-R loop (``render.mesh.prepare_vertices``,
``render.mesh.texture_mapping``, ``metrics.render.mask_iou``), lighting and deferred shading
(``render.lighting``, ``render.easy_render``), and the mesh Laplacian regulariser of the loss
(``ops.mesh.{adjacency_matrix, uniform_laplacian, average_face_vertex_features,
compute_vertex_normals}``, ``metrics.trianglemesh.uniform_laplacian_smoothing``, and
``ops.mesh.UniformLaplacian``, which applies the Laplacian without its V x V matrix), Loop
subdivision (``ops.mesh.subdivide_trianglemesh`` and ``ops.mesh.LoopSubdivision``, which builds its
levels once), and DMTet's tet-grid operators (``ops.conversions.marching_tetrahedra``,
``ops.conversions.MarchingTetrahedra``, which builds the grid's topology once, and
``ops.mesh.subdivide_tetmesh``), and the point-in-mesh test (``ops.mesh.check_sign``,
``ops.mesh.CheckSign``, which builds the mesh once, and ``_C.ops.mesh.unbatched_mesh_intersection_cuda``),
and marching cubes (``ops.conversions.voxelgrids_to_trianglemeshes``, every view in one call, and
``_C.ops.conversions.unbatched_mcube_forward_cuda``), and cubic meshes from voxel grids
(``ops.conversions.voxelgrids_to_cubic_meshes``, every view in one call), and the point-to-mesh distance
(``metrics.trianglemesh.point_to_mesh_distance``, every view in one call, and ``_C.metrics``),
and the voxel-grid operators (``ops.voxelgrid.{fill, extract_surface, extract_odms, project_odms,
downsample}``, every view in one launch per kernel), and farthest point sampling
(``ops.pointcloud.farthest_point_sampling``, deterministic, every view in one call, with
``ops.pointcloud.center_points``); see DESIGN.md for scope.  There is no CPU fallback: every entry point
raises if the CUDA library (kaolin_b200/csrc, built in-tree) is missing or the
tensors are not on a CUDA device.
"""
__version__ = "0.1.0"

from . import render   # noqa: E402,F401
from . import metrics  # noqa: E402,F401
from . import ops      # noqa: E402,F401
from . import _C       # noqa: E402,F401
