from . import render  # noqa: F401
from . import trianglemesh  # noqa: F401
from .trianglemesh import point_to_mesh_distance  # noqa: F401
