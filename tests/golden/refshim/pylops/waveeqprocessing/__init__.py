from . import kirchhoff, lsm  # noqa: F401
from .kirchhoff import Kirchhoff  # noqa: F401
from .lsm import LSM  # noqa: F401
