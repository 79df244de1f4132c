"""Restatement of the part of third-party pylops' operator algebra that tutorials/poststack.py uses -- TEST
INFRASTRUCTURE for tests/golden/make_golden_poststack.py: ``Op.H`` (adjoint), ``Op1 * Op2`` / ``Op1 @ Op2``
(product) and ``Op @ x`` (matvec).  Operators that take part derive from :class:`AlgebraOperator`; the products and
adjoints it builds do too."""
import numpy as np

from . import LinearOperator


class AlgebraOperator(LinearOperator):
    @property
    def H(self):
        return AdjointLinearOperator(self)

    def __matmul__(self, other):
        if isinstance(other, LinearOperator):
            return ProductLinearOperator(self, other)
        return self.matvec(other)

    __mul__ = __matmul__


class AdjointLinearOperator(AlgebraOperator):
    def __init__(self, A):
        self.A = A
        super().__init__(dtype=A.dtype, shape=(A.shape[1], A.shape[0]))

    def _matvec(self, x):
        return self.A.rmatvec(x)

    def _rmatvec(self, x):
        return self.A.matvec(x)


class ProductLinearOperator(AlgebraOperator):
    def __init__(self, A, B):
        assert A.shape[1] == B.shape[0]
        self.A, self.B = A, B
        super().__init__(dtype=np.result_type(A.dtype, B.dtype), shape=(A.shape[0], B.shape[1]))

    def _matvec(self, x):
        return self.A.matvec(self.B.matvec(x))

    def _rmatvec(self, x):
        return self.B.rmatvec(self.A.rmatvec(x))
