from . import mesh  # noqa: F401
from . import easy_render  # noqa: F401
from . import lighting  # noqa: F401
