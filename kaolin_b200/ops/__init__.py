"""kaolin.ops drop-ins: the mesh Laplacian, adjacency, vertex averaging, Loop subdivision, tet-mesh
subdivision and marching tetrahedra on sm_90a kernels."""
from . import mesh  # noqa: F401
from . import conversions  # noqa: F401
