"""kaolin.ops drop-ins: the mesh Laplacian, adjacency and vertex averaging on sm_90a kernels."""
from . import mesh  # noqa: F401
