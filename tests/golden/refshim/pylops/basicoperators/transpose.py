"""Restatement of third-party ``pylops.basicoperators.Transpose`` -- TEST INFRASTRUCTURE for
tests/golden/make_golden_poststack.py (imported as ``pylops.basicoperators.transpose``)."""
import numpy as np

from .._algebra import AlgebraOperator


class Transpose(AlgebraOperator):
    """Restatement of third-party ``pylops.basicoperators.Transpose`` (pylops 2.x): ``x.reshape(dims)
    .transpose(axes).ravel()``, adjoint with the inverse permutation ``argsort(axes)`` on ``dims[axes]``."""

    def __init__(self, dims, axes, dtype="float64"):
        self.dims = tuple(int(d) for d in dims)
        self.axes = tuple(int(a) for a in axes)
        if sorted(self.axes) != list(range(len(self.dims))):
            raise ValueError("axes must be a permutation of range(len(dims))")
        self.dimsd = tuple(self.dims[a] for a in self.axes)
        self.axesd = tuple(int(a) for a in np.argsort(self.axes))
        n = int(np.prod(self.dims))
        super().__init__(dtype=np.dtype(dtype), shape=(n, n))

    def _matvec(self, x):
        return np.reshape(x, self.dims).transpose(self.axes).ravel()

    def _rmatvec(self, x):
        return np.reshape(x, self.dimsd).transpose(self.axesd).ravel()
