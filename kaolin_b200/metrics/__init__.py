from . import render  # noqa: F401
from . import trianglemesh  # noqa: F401
