"""Restatement of third-party ``pylops.basicoperators.MatrixMult`` with ``otherdims`` -- TEST INFRASTRUCTURE for the
2-D wavelet branch of post-stack modelling (refshim/pylops/avo/poststack_nonstationary.py).  The dense block without
``otherdims`` that the reference's hot path uses is ``pylops.MatrixMult`` (refshim/pylops/__init__.py)."""
import numpy as np

from .. import LinearOperator


class MatrixMult(LinearOperator):
    """pylops 2.x ``MatrixMult(A, otherdims)``: x is a ``(A.shape[1],) + otherdims`` array and ``A`` acts on its first
    axis, ``y = (A @ x.reshape(A.shape[1], -1)).ravel()``; the adjoint applies ``A^H`` the same way"""

    def __init__(self, A, otherdims=None, dtype="float64"):
        self.A = A
        self.otherdims = () if otherdims is None else tuple(int(d) for d in np.atleast_1d(otherdims))
        nother = int(np.prod(self.otherdims))
        super().__init__(dtype=np.dtype(dtype), shape=(A.shape[0] * nother, A.shape[1] * nother))

    def _matvec(self, x):
        return (self.A @ np.reshape(x, (self.A.shape[1], -1))).ravel()

    def _rmatvec(self, x):
        return (self.A.conj().T @ np.reshape(x, (self.A.shape[0], -1))).ravel()
