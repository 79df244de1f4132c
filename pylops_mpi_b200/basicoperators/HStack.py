"""``MPIHStack`` = adjoint of an ``MPIVStack`` of adjoints
(pylops_mpi/basicoperators/HStack.py:90-106)."""
from __future__ import annotations

from typing import Sequence

from ..comm import COMM_WORLD
from ..LinearOperator import MPILinearOperator
from ..local import _LocalAdjoint
from .VStack import MPIVStack


class MPIHStack(MPILinearOperator):
    def __init__(self, ops: Sequence, base_comm=COMM_WORLD, dtype=None):
        self.ops = ops
        hops = [_LocalAdjoint(op) for op in ops]
        self.HStack = MPIVStack(ops=hops, base_comm=base_comm, dtype=dtype).H
        super().__init__(shape=self.HStack.shape, dtype=self.HStack.dtype, base_comm=base_comm)

    def _matvec(self, x):
        return self.HStack.matvec(x)

    def _rmatvec(self, x):
        return self.HStack.rmatvec(x)
