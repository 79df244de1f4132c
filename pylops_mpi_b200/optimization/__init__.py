from .basic import cg, cgls, lsqr  # noqa: F401
from .cls_basic import CG, CGLS, LSQR  # noqa: F401
from .sparsity import ista, fista  # noqa: F401
from .cls_sparsity import ISTA, FISTA  # noqa: F401
from .eigs import power_iteration  # noqa: F401
