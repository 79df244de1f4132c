"""Functional wrappers ``cg`` / ``cgls`` (pylops_mpi/optimization/basic.py:13-148) and ``lsqr`` (pylops 2.x's
signature; an extension, the reference has no LSQR)."""
from __future__ import annotations

from typing import Callable, Optional, Tuple

from ..DistributedArray import DistributedArray
from .cls_basic import CG, CGLS, LSQR


def cg(Op, y, x0: Optional[DistributedArray] = None, niter: int = 10, tol: float = 1e-4,
       show: bool = False, itershow: Tuple[int, int, int] = (10, 10, 10),
       callback: Optional[Callable] = None):
    cgsolve = CG(Op)
    if callback is not None:
        cgsolve.callback = callback
    x, iiter, cost = cgsolve.solve(y=y, x0=x0, tol=tol, niter=niter, show=show, itershow=itershow)
    return x, iiter, cost


def cgls(Op, y, x0: Optional[DistributedArray] = None, niter: int = 10, damp: float = 0.0,
         tol: float = 1e-4, show: bool = False, itershow: Tuple[int, int, int] = (10, 10, 10),
         callback: Optional[Callable] = None):
    cgsolve = CGLS(Op)
    if callback is not None:
        cgsolve.callback = callback
    x, istop, iiter, r1norm, r2norm, cost = cgsolve.solve(y=y, x0=x0, niter=niter, damp=damp,
                                                          tol=tol, show=show, itershow=itershow)
    return x, istop, iiter, r1norm, r2norm, cost


def lsqr(Op, y, x0: Optional[DistributedArray] = None, damp: float = 0.0, atol: float = 1e-8, btol: float = 1e-8,
         conlim: float = 1e8, niter: int = 10, calc_var: bool = True, show: bool = False,
         itershow: Tuple[int, int, int] = (10, 10, 10), callback: Optional[Callable] = None):
    """LSQR as pylops 2.x's ``lsqr``: returns ``(x, istop, iiter, r1norm, r2norm, anorm, acond, arnorm, xnorm, var,
    cost)`` with ``cost`` the r1norm history (initial value, then one entry per iteration).  The scalars, ``istop``
    and ``var`` are those of ``scipy.sparse.linalg.lsqr(..., iter_lim=niter)`` with the same parameters."""
    lsqrsolve = LSQR(Op)
    if callback is not None:
        lsqrsolve.callback = callback
    return lsqrsolve.solve(y=y, x0=x0, damp=damp, atol=atol, btol=btol, conlim=conlim, niter=niter,
                           calc_var=calc_var, show=show, itershow=itershow)
