"""kaolin.ops drop-ins: the mesh Laplacian, adjacency, vertex averaging and Loop subdivision on sm_90a
kernels."""
from . import mesh  # noqa: F401
