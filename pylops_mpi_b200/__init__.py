"""pylops_mpi_b200 -- H100-native (sm_90a CUDA + NCCL/NVLink) implementation of
the pylops-mpi distributed matvec / rmatvec hot path, behind the reference's
own operator API (``DistributedArray``, ``MPILinearOperator`` and the
BlockDiag / VStack / MatrixMult / FirstDerivative / Fredholm1 operators,
``cgls``, ``dottest``).  Importing the package loads ``libb200lops.so``; there
is no CPU fallback.
"""
from . import _lib  # noqa: F401  (raises if the CUDA extension is missing)
from .comm import Comm, COMM_WORLD, get_comm_world  # noqa: F401
from .DistributedArray import DistributedArray, Partition, local_split, subcomm_split  # noqa: F401
from .LinearOperator import MPILinearOperator, asmpilinearoperator  # noqa: F401
from .basicoperators import *  # noqa: F401,F403
from .signalprocessing import *  # noqa: F401,F403
from . import waveeqprocessing  # noqa: F401
from .waveeqprocessing import MPIMDC  # noqa: F401
from .StackedArray import StackedDistributedArray  # noqa: F401
from .StackedLinearOperator import MPIStackedLinearOperator  # noqa: F401
from .basicoperators import MPIStackedBlockDiag, MPIStackedVStack, MPIGradient  # noqa: F401
from .optimization.basic import cg, cgls, lsqr  # noqa: F401
from .optimization.cls_basic import CG, CGLS, LSQR  # noqa: F401
from .optimization.sparsity import ista, fista  # noqa: F401
from .optimization.cls_sparsity import ISTA, FISTA  # noqa: F401
from .optimization.eigs import power_iteration  # noqa: F401
from .utils.dottest import dottest  # noqa: F401
from . import local  # noqa: F401
from .local import MatrixMult  # noqa: F401

__version__ = "0.1.0"
