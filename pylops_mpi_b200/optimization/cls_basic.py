"""CG / CGLS solvers with the reference's recurrences, stopping rule and
outputs (pylops_mpi/optimization/cls_basic.py:12-531); the ``Solver`` base the
reference takes from pylops (callbacks, timing, banner) is restated minimally.

Two execution modes, same numbers:
  * generic: the reference's exact sequence of DistributedArray operations;
  * fused (default on device arrays): identical recurrences, but axpy-style
    updates run in place (no temporaries), the reductions they feed are fused
    into them and the step scalars stay on the device.  CGLS has ONE fused
    iteration (``CGLS._body``): ``step()`` runs it eagerly and reads its
    scalars with one host synchronisation, ``run()`` replays it as a CUDA
    graph and reads them once per block, so every mode gives the same bits.
    LSQR (an extension: the reference has none) is built the same way.
"""
from __future__ import annotations

import sys
import time
from typing import List, Optional, Sequence

import numpy as np
import torch

from .. import _lib
from ..Distributed import allreduce_
from ..DistributedArray import DistributedArray
from ..local import _KernelOperator
from ..utils.partition import local_split_sizes, offsets
from .lsqr_host import (_AA, _ALFA, _ATOL, _BB, _BETA, _BNORM, _BTOL, _CS2, _CTOL, _CUB, _CVA, _CVB, _DAMP,
                        _DAMPSQ, _DD, _INV_ALFA, _INV_RHO, _ITER_LIM, _ITN, _NHIST, _NSTATE, _PHIBAR, _RHOBAR,
                        _SCRATCH, _STOPPED, _T1, _T2, lsqr_scalars_host)


class Solver:
    """subset of pylops.optimization.basesolver.Solver used by CG/CGLS"""

    def __init__(self, Op, callbacks: Optional[Sequence] = None):
        self.Op = Op
        self.callbacks = callbacks
        self.tstart = time.time()

    def callback(self, x, *args, **kwargs):
        pass

    def _print_solver(self, text: str = "", nbar: int = 80) -> None:
        print(f"{type(self).__name__}" + text)
        print("-" * nbar + "\n" + f"The Operator Op has {self.Op.shape[0]} rows and {self.Op.shape[1]} cols")

    def _print_finalize(self, nbar: int = 80) -> None:
        print(f"\nIterations = {self.iiter}        Total time (s) = {self.telapsed:.2f}")
        print("-" * nbar + "\n")


_GRAPH_SAFE_TYPES = ("MPIBlockDiag", "MPIVStack", "MPIHStack", "MPIFirstDerivative", "MPISecondDerivative",
                     "_MPISummaMatrixMult", "_MPIBlockMatrixMult", "_AdjointLinearOperator", "_TransposedLinearOperator",
                     "_ProductLinearOperator", "_ScaledLinearOperator", "_SumLinearOperator", "_ConjLinearOperator")


_GRAPH_POOL = {}


def _graph_pool():
    """process-wide (per device) memory pool shared by every solver capture.  torch only lets a capture join an
    existing pool while at least one live graph still references it (otherwise capture_begin trips
    'use_count > 0' in the caching allocator -- seen when one solver's graph had been freed before the next solver
    captured), so a tiny ANCHOR graph captured once per device owns the pool for the life of the process."""
    dev = torch.cuda.current_device()
    hit = _GRAPH_POOL.get(dev)
    if hit is None:
        torch.zeros(16, device="cuda")                   # load the fill kernel outside any capture
        g = torch.cuda.CUDAGraph()
        main = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(main)
        with torch.cuda.stream(side):
            g.capture_begin(capture_error_mode="thread_local")
            try:
                keep = torch.zeros(16, device="cuda")    # one allocation + one kernel node: the graph is not empty
            finally:
                g.capture_end()
        main.wait_stream(side)
        hit = _GRAPH_POOL[dev] = (g.pool(), g, keep)
    return hit[0]


def _reset_capture_state():
    """a capture that died half-way leaves torch's CUDA generator flagged as 'capturing' (every later RNG call then
    raises 'Offset increment outside graph capture'): one empty, successful capture clears the flag"""
    try:
        g = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            g.capture_begin(capture_error_mode="thread_local")
            g.capture_end()
        torch.cuda.synchronize()
    except Exception:
        pass


def _graph_safe(Op) -> bool:
    """may an apply of ``Op`` be captured once in a CUDA graph and replayed?  Conservative whitelist: operators of
    this package whose apply is a fixed sequence of kernel launches / collectives with no host-side per-call state,
    the rank-local kernel operators by type, the others by name (MPIFredholm1's fused mode toggles double buffers on
    the host, third-party operators are unknown -> eager)"""
    if isinstance(Op, _KernelOperator):
        return True
    name = type(Op).__name__
    if name not in _GRAPH_SAFE_TYPES:
        return False
    if name == "_MPISummaMatrixMult" and Op.base_comm.Get_size() > 1 and not getattr(Op, "_stationary", False):
        return False       # the pipelined SUMMA forks streams per round: keep it eager
    for child in list(getattr(Op, "args", ())) + list(getattr(Op, "ops", ())):
        if hasattr(child, "shape") and not isinstance(child, (int, float, complex, np.number)):
            if not _graph_safe(child):
                return False
    return True


def _generic(*arrs) -> bool:
    """True when any operand is not a plain DistributedArray (StackedDistributedArray models / data,
    test_solver.py:303+): the solvers then run the reference's own sequence of ``dot / + / *`` operations
    instead of the fused device-scalar step"""
    return any(not isinstance(a, DistributedArray) for a in arrs)


def _absdot(a: DistributedArray, b: DistributedArray) -> float:
    """|a . conj(b)| as the reference computes it (np.abs(a.dot(b.conj())).item())"""
    return float(np.abs(a.dot(b.conj())).item())


def _self_dots(arrs: Sequence[DistributedArray]) -> List[float]:
    """[|a . conj(a)| for a in arrs] in ONE kernel launch + ONE Allreduce + ONE host sync"""
    k = len(arrs)
    views = [a._scatter_view() for a in arrs]
    same = all(v.numel() == views[0].numel() and v.dtype == views[0].dtype for v in views) and \
        all(a.sub_comm is arrs[0].sub_comm for a in arrs)
    if not same or k > 4:
        return [_absdot(a, a) for a in arrs]
    out = torch.zeros(2 * k, dtype=torch.float64, device=views[0].device)
    _dots_device(arrs, out)
    allreduce_(arrs[0].sub_comm, out, "sum")
    res = out.cpu().numpy()
    if views[0].dtype.is_complex:
        return [float(np.abs(complex(res[2 * i], res[2 * i + 1]))) for i in range(k)]
    return [float(np.abs(res[i])) for i in range(k)]


def _dots_device(arrs: Sequence[DistributedArray], out: torch.Tensor, offset: int = 0) -> int:
    """out[offset + i*stride] = a_i . conj(a_i) (LOCAL partial sums, float64, no host sync);
    returns the number of doubles written.  One launch when all arrays share a length."""
    import ctypes as C
    views = [a._scatter_view() for a in arrs]
    stride = 2 if views[0].dtype.is_complex else 1
    n0 = views[0].numel()
    if all(v.numel() == n0 for v in views) and len(views) <= 4:
        groups = [views]
    else:
        groups = [[v] for v in views]
    off = offset
    for g in groups:
        k = len(g)
        n = g[0].numel()
        ptrs = (C.c_void_p * k)(*[v.data_ptr() if n else None for v in g])
        _lib.check(_lib.lib.b2_dot_multi(_lib.ctx(), k, ptrs, ptrs, n, _lib.code(g[0].dtype), 1,
                                         out.data_ptr() + 8 * off, _lib.stream()), "b2_dot_multi")
        off += k * stride
    return off - offset


def _scalar_div(out: torch.Tensor, oi: int, num: torch.Tensor, ni: int, den1: torch.Tensor, d1: int,
                den2: Optional[torch.Tensor] = None, d2: int = 0, alpha: float = 0.0):
    """out[oi] = |num[ni] / (den1[d1] + alpha * den2[d2])| on the device"""
    _lib.check(_lib.lib.b2_scalar_div(out.data_ptr() + 8 * oi, num.data_ptr() + 8 * ni, den1.data_ptr() + 8 * d1,
                                      (den2.data_ptr() + 8 * d2) if den2 is not None else None, float(alpha),
                                      _lib.stream()), "b2_scalar_div")


def _lincomb_dev(out: DistributedArray, a_dev: Optional[torch.Tensor], ai: int, a_scale: float,
                 x: DistributedArray, b_dev: Optional[torch.Tensor], bi: int, b_scale: float,
                 y: DistributedArray):
    """out = (a_scale * a_dev[ai]) * x + (b_scale * b_dev[bi]) * y with DEVICE scalars (NULL -> 1)"""
    o, xv, yv = out._cont(), out._as_mine(x), out._as_mine(y)   # one dtype for the kernel: the updated array's
    n = o.numel()
    if n:
        _lib.check(_lib.lib.b2_lincomb_dev(_lib.ctx(), o.data_ptr(),
                                           (a_dev.data_ptr() + 8 * ai) if a_dev is not None else None, float(a_scale),
                                           xv.data_ptr(),
                                           (b_dev.data_ptr() + 8 * bi) if b_dev is not None else None, float(b_scale),
                                           yv.data_ptr(), n, _lib.code(o.dtype), _lib.stream()), "b2_lincomb_dev")
    if o is not out.local_array:
        out.local_array.copy_(o)


def _lincomb_dev_norm2(out: DistributedArray, a_dev: Optional[torch.Tensor], ai: int, a_scale: float,
                       x: DistributedArray, b_dev: Optional[torch.Tensor], bi: int, b_scale: float,
                       y: DistributedArray, dev: torch.Tensor, slot: int) -> bool:
    """out = (a_scale a_dev[ai]) x + (b_scale b_dev[bi]) y AND dev[slot] = sum |out|^2 (local partial) in ONE kernel.
    Falls back (returns False after doing the plain update) for BROADCAST arrays -- their reduction runs on the
    re-scattered view -- and mixed dtypes."""
    from ..DistributedArray import Partition
    o = out._cont()
    fusable = out.partition is Partition.SCATTER and o is out.local_array and \
        x._tdtype == out._tdtype and y._tdtype == out._tdtype and out._tdtype in (torch.float32, torch.float64,
                                                                                 torch.complex64, torch.complex128)
    if not fusable:
        _lincomb_dev(out, a_dev, ai, a_scale, x, b_dev, bi, b_scale, y)
        return False
    _lib.check(_lib.lib.b2_lincomb_dev_norm2(_lib.ctx(), o.data_ptr(),
                                             (a_dev.data_ptr() + 8 * ai) if a_dev is not None else None, float(a_scale),
                                             x._cont().data_ptr(),
                                             (b_dev.data_ptr() + 8 * bi) if b_dev is not None else None, float(b_scale),
                                             y._cont().data_ptr(), o.numel(), _lib.code(o.dtype),
                                             dev.data_ptr() + 8 * slot, _lib.stream()), "b2_lincomb_dev_norm2")
    return True


class CG(Solver):
    """cls_basic.py:12-249"""

    def setup(self, y, x0, niter: Optional[int] = None, tol: float = 1e-4, show: bool = False):
        self.y = y
        self.niter = niter
        self.tol = tol
        x = x0.copy()
        self.r = self.y - self.Op.matvec(x)
        self.rank = x.rank
        self.c = self.r.copy()
        self._gen = _generic(x, self.r)
        self.kold = _absdot(self.r, self.r) if self._gen else _self_dots([self.r])[0]
        self.cost: List = [float(np.sqrt(self.kold))]
        self.iiter = 0
        return x

    def _step_generic(self, x):
        """cls_basic.py:127-141 verbatim in operations (stacked arrays)"""
        Opc = self.Op.matvec(self.c)
        cOpc = np.abs(self.c.dot(Opc.conj()))
        a = float((self.kold / cOpc).item())
        x += a * self.c
        self.r -= a * Opc
        k = _absdot(self.r, self.r)
        b = float(k / self.kold)
        self.c = self.r + b * self.c
        self.kold = k
        self.iiter += 1
        self.cost.append(float(np.sqrt(self.kold)))
        return x

    def step(self, x, show: bool = False):
        if self._gen:
            return self._step_generic(x)
        Opc = self.Op.matvec(self.c)
        cOpc = np.abs(self.c.dot(Opc.conj()))
        with np.errstate(divide="ignore", invalid="ignore"):      # the reference divides NumPy scalars: inf / nan, no raise
            a = float((np.float64(self.kold) / cOpc).item())
        x.axpy_(a, self.c)
        self.r.axpy_(-a, Opc)
        k = _self_dots([self.r])[0]
        b = float(k / self.kold)
        self.c.xpby_(self.r, b)
        self.kold = k
        self.iiter += 1
        self.cost.append(float(np.sqrt(self.kold)))
        return x

    def run(self, x, niter: Optional[int] = None, show: bool = False, itershow=(10, 10, 10)):
        niter = self.niter if niter is None else niter
        if niter is None:
            raise ValueError("niter must not be None")
        while self.iiter < niter and self.kold > self.tol:
            x = self.step(x, False)
            self.callback(x)
        return x

    def finalize(self, show: bool = False) -> None:
        self.tend = time.time()
        self.telapsed = self.tend - self.tstart
        self.cost = np.array(self.cost)

    def solve(self, y, x0, niter: int = 10, tol: float = 1e-4, show: bool = False,
              itershow=(10, 10, 10)):
        x = self.setup(y=y, x0=x0, niter=niter, tol=tol, show=show)
        x = self.run(x, niter, show=show, itershow=itershow)
        self.finalize(show)
        return x, self.iiter, self.cost


class _DeviceLoopSolver(Solver):
    """a solver with ONE fused device iteration ``_body(*args)`` (no host synchronisation inside): ``_iterate`` runs
    the first iteration of a block run eagerly, then captures the body once as a CUDA graph and replays it"""

    def _iterate(self, *args):
        """one iteration of a block run: the first runs eagerly (every kernel of the body gets loaded, lazy
        workspaces and communicators exist), then the body is captured once as a CUDA graph and replayed"""
        if self._graph is None and self._capture and self._warm:
            t_cap = time.perf_counter()
            try:
                # manual capture on a side stream (torch.cuda.graph() would add a device synchronise, a
                # gc.collect() and an empty_cache() -- milliseconds, comparable to a whole 50-iteration solve)
                pool = _graph_pool()
                t_pool = time.perf_counter()
                g = torch.cuda.CUDAGraph()
                main = torch.cuda.current_stream()
                side = torch.cuda.Stream()
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    # one process-wide memory pool for all captures: the temporaries of the first capture are
                    # cudaMalloc'ed (slow when peers have this device mapped: measured 3.1 ms at 2 GPUs vs 0.65 ms
                    # at 1), later captures reuse the cached blocks
                    # thread_local error mode: NCCL's helper threads keep polling CUDA while we capture
                    # (observed at 8 ranks: a "global"-mode capture was invalidated and left torch's RNG state
                    # stuck in capture mode)
                    g.capture_begin(pool=pool, capture_error_mode="thread_local")   # records only
                    t_begin = time.perf_counter()
                    try:
                        self._body(*args)
                    finally:
                        t_body = time.perf_counter()
                        g.capture_end()
                main.wait_stream(side)
                self._graph = g
                t_end = time.perf_counter()
                self.graph_capture_ms = (t_end - t_cap) * 1e3
                self.graph_capture_breakdown_ms = {"pool": (t_pool - t_cap) * 1e3, "begin": (t_begin - t_pool) * 1e3,
                                                   "body": (t_body - t_begin) * 1e3, "end": (t_end - t_body) * 1e3}
            except Exception as exc:               # not capturable (host sync inside an operator ...): stay eager
                self._capture = False
                self.graph_error = repr(exc)[:300]
                print(f"[b200 {type(self).__name__.lower()}] CUDA-graph capture failed, running eagerly: "
                      f"{self.graph_error}", file=sys.stderr)
                torch.cuda.synchronize()
                _reset_capture_state()
        if self._graph is not None:
            self._graph.replay()
            self.graph_replays += 1
        else:
            self._body(*args)
            self._warm = True

    def _start_blocks(self):
        self._graph, self._warm, self._capture = None, False, _graph_safe(self.Op)
        self.graph_replays, self.graph_error = 0, (None if self._capture else "operator not on the graph-safe list")

    def _plain_callback(self) -> bool:
        """no callback to call per iteration: neither overridden in a subclass nor set on the instance
        (cgls(callback=...)) nor given as ``callbacks``"""
        return type(self).callback is Solver.callback and "callback" not in vars(self) and not self.callbacks


class CGLS(_DeviceLoopSolver):
    """cls_basic.py:252-531"""

    def _print_step(self, x) -> None:
        x0 = (x if isinstance(x, DistributedArray) else x[0]).local_array.reshape(-1)[0].item()
        strx = f"{x0:1.2e}   " if isinstance(x0, complex) else f"{x0:11.4e}        "
        print(f"{self.iiter:6g}       " + strx + f"{self.cost[self.iiter]:11.4e}    {self.cost1[self.iiter]:11.4e}")
        sys.stdout.flush()

    def setup(self, y, x0, niter: Optional[int] = None, damp: float = 0.0, tol: float = 1e-4,
              show: bool = False):
        self.y = y
        self.damp = damp ** 2
        self.tol = tol
        self.niter = niter
        x = x0.copy()
        self.s = self.y - self.Op.matvec(x)
        self._gen = _generic(x, self.s)
        if self._gen:
            return self._setup_generic(x, damp, show)
        r = self.Op.rmatvec(self.s)
        if damp != 0.0:
            r.axpy_(-damp, x)                       # r = Op^H s - damp * x   (:341-342)
        self.rank = x.rank
        self.c = r.copy()
        self.kold = _self_dots([r])[0]
        self._st = 2 if (x._tdtype.is_complex or self.s._tdtype.is_complex or self.c._tdtype.is_complex) else 1
        self._dev = torch.zeros(16, dtype=torch.float64, device=x.local_array.device)
        self._dev[self._slots()[-1]] = self.kold
        self._cc_ready = False                      # the first body computes c.c itself
        self.cost = []
        self.cost1 = []
        ss, xx = _self_dots([self.s, x]) if self.s.local_shape == x.local_shape else \
            (_self_dots([self.s])[0], _self_dots([x])[0])
        self.cost.append(float(np.sqrt(ss)))
        # note: un-squared damp here, squared in step(), as in the reference (:358 vs :401)
        self.cost1.append(np.sqrt(float(self.cost[0] ** 2 + damp * xx)))
        self.iiter = 0
        if show and self.rank == 0:
            self._print_solver(nbar=65)
            print(f"damp = {self.damp:10e}\ttol = {self.tol:10e}\tniter = {self.niter}")
            print("-" * 65 + "\n")
            print("    Itn          x[0]              r1norm         r2norm")
        return x

    def _setup_generic(self, x, damp, show):
        """cls_basic.py:339-366 in the reference's own operations (stacked arrays)"""
        r = self.Op.rmatvec(self.s) - x * damp
        self.rank = x.rank
        self.c = r.copy()
        self.q = self.Op.matvec(self.c)
        self.kold = _absdot(r, r)
        self.cost = [float(self.s.norm().item())]
        self.cost1 = [np.sqrt(float(self.cost[0] ** 2 + damp * _absdot(x, x)))]
        self.iiter = 0
        if show and self.rank == 0:
            self._print_solver(nbar=65)
            print(f"damp = {self.damp:10e}\ttol = {self.tol:10e}\tniter = {self.niter}")
            print("-" * 65 + "\n")
            print("    Itn          x[0]              r1norm         r2norm")
        return x

    def _step_generic(self, x, show):
        """cls_basic.py:389-404 verbatim in operations"""
        a = float(np.abs(self.kold / (self.q.dot(self.q.conj()) + self.damp * self.c.dot(self.c.conj()))).item())
        x += a * self.c
        self.s -= a * self.q
        r = self.Op.rmatvec(self.s) - self.damp * x
        k = _absdot(r, r)
        b = float(k / self.kold)
        self.c = r + b * self.c
        self.q = self.Op.matvec(self.c)
        self.kold = k
        self.iiter += 1
        self.cost.append(float(self.s.norm().item()))
        self.cost1.append(np.sqrt(float(self.cost[self.iiter] ** 2 + self.damp * _absdot(x, x))))
        if show and self.rank == 0:
            self._print_step(x)
        return x

    def step(self, x, show: bool = False):
        """One CGLS iteration (cls_basic.py:370-404): the fused body run eagerly, 2 Allreduces and ONE host
        synchronisation (the reference: 5 and 5)."""
        if self._gen:
            return self._step_generic(x, show)
        hist = torch.empty((1, 3), dtype=torch.float64, device=self._dev.device)
        self._body(x, hist, torch.zeros(1, dtype=torch.int64, device=hist.device))
        self._absorb(hist[0].cpu().numpy())
        if show and self.rank == 0:
            self._print_step(x)
        return x

    def _slots(self):
        """offsets in ``_dev`` of the fused iteration's scalars [q.q, c.c | k, s.s, x.x | a, b | kold]; dots take
        (re, im) pairs as soon as ANY of the arrays is complex (a real model with complex-typed data, as in MPIMDC,
        must not let a complex dot spill into its neighbour's slot)"""
        st = self._st
        return 0, st, 4, 4 + st, 4 + 2 * st, 12, 13, 14

    def _absorb(self, row) -> None:
        """host-side bookkeeping of one iteration from its history row (k, s.s, x.x)"""
        k, ss, xx = row
        self.kold = float(k)
        self.iiter += 1
        self.cost.append(float(np.sqrt(ss)))
        self.cost1.append(np.sqrt(float(self.cost[self.iiter] ** 2 + self.damp * xx)))

    def _body(self, x, hist: torch.Tensor, it_dev: torch.Tensor):
        """one CGLS iteration in ROTATED order (q = Op c first): every array that crosses iterations (x, s, c) is
        updated in place and q, r live and die inside the body, so a captured graph can be replayed verbatim.  No
        host synchronisation: the three per-iteration scalars go to ``hist[it_dev]``."""
        dev, st = self._dev, self._st
        QQ, CC, K, SS, XX, A_, B_, KOLD = self._slots()
        sub = self.c.sub_comm
        q = self.Op.matvec(self.c)
        _dots_device([q], dev, QQ)
        if not self._cc_ready:                      # c.c normally comes fused with the update of c (end of the body)
            _dots_device([self.c], dev, CC)
        allreduce_(sub, dev[0:2 * st], "sum")
        _scalar_div(dev, A_, dev, KOLD, dev, QQ, dev, CC, self.damp)
        # x += a c (+ x.x), s -= a q (+ s.s): update and the reduction the cost needs, one pass each
        if not _lincomb_dev_norm2(x, dev, A_, 1.0, self.c, None, 0, 1.0, x, dev, XX):
            _dots_device([x], dev, XX)
        if not _lincomb_dev_norm2(self.s, dev, A_, -1.0, q, None, 0, 1.0, self.s, dev, SS):
            _dots_device([self.s], dev, SS)
        r = self.Op.rmatvec(self.s)
        if self.damp != 0.0:
            r.axpy_(-self.damp, x)
        _dots_device([r], dev, K)
        allreduce_(sub, dev[4:4 + 3 * st], "sum")
        _scalar_div(dev, B_, dev, K, dev, KOLD)
        # c = r + b c (+ c.c for the next iteration's step length)
        self._cc_ready = _lincomb_dev_norm2(self.c, None, 0, 1.0, r, dev, B_, 1.0, self.c, dev, CC)
        _lib.check(_lib.lib.b2_history_push(dev.data_ptr() + 8 * K, 3, st, hist.data_ptr(), it_dev.data_ptr(),
                                            hist.shape[0], dev.data_ptr() + 8 * KOLD, dev.data_ptr() + 8 * K,
                                            _lib.stream()), "b2_history_push")

    def _run_blocks(self, x, niter: int):
        """remaining iterations in blocks of :meth:`_iterate`; the host reads the scalar history once per block.
        With tol > 0 a block is at most 8 iterations and is re-run from a checkpoint up to the stopping iteration,
        so x, cost and the iteration count are exactly those of the reference's per-iteration test ``kold > tol``
        (cls_basic.py:436)."""
        device = x.local_array.device
        it0 = self.iiter
        hist = torch.zeros((niter - it0 + 2, 3), dtype=torch.float64, device=device)
        it_dev = torch.zeros(1, dtype=torch.int64, device=device)
        self._start_blocks()
        block = niter - it0 if self.tol <= 0.0 else 8
        while self.iiter < niter and self.kold > self.tol:
            n = min(block, niter - self.iiter)
            start = self.iiter - it0
            live = (x.local_array, self.s.local_array, self.c.local_array, self._dev)
            ckpt, cc_ready = [a.clone() for a in live], self._cc_ready
            for _ in range(n):
                self._iterate(x, hist, it_dev)
            for i, row in enumerate(hist[start:start + n].cpu().numpy()):
                self._absorb(row)
                if not (self.iiter < niter and self.kold > self.tol):
                    break
            if i + 1 < n:
                # the stopping test fired inside the block: redo exactly the iterations up to it from the checkpoint
                for dst, src in zip(live, ckpt):
                    dst.copy_(src)
                it_dev.fill_(start)
                if self._cc_ready and not cc_ready:     # c.c of the restored c, as the first body computed it
                    _dots_device([self.c], self._dev, self._slots()[1])
                for _ in range(i + 1):
                    self._iterate(x, hist, it_dev)
            del ckpt
        self._graph = None
        return x

    def run(self, x, niter: Optional[int] = None, show: bool = False, itershow=(10, 10, 10)):
        niter = self.niter if niter is None else niter
        if niter is None:
            raise ValueError("niter must not be None")
        # a callback, overridden in a subclass or set on the instance (cgls(callback=...)), sees every iteration
        if not self._gen and not show and self._plain_callback() and niter - self.iiter > 0:
            return self._run_blocks(x, niter)
        while self.iiter < niter and self.kold > self.tol:
            showstep = bool(show and (self.iiter < itershow[0] or niter - self.iiter < itershow[1]
                                      or self.iiter % itershow[2] == 0))
            x = self.step(x, showstep)
            self.callback(x)
        return x

    def finalize(self, show: bool = False, **kwargs) -> None:
        self.tend = time.time()
        self.telapsed = self.tend - self.tstart
        self.istop = 1 if self.kold < self.tol else 2
        self.r1norm = self.kold
        self.r2norm = self.cost1[self.iiter]
        if show and self.rank == 0:
            self._print_finalize(nbar=65)
        self.cost = np.array(self.cost)

    def solve(self, y, x0, niter: int = 10, damp: float = 0.0, tol: float = 1e-4, show: bool = False,
              itershow=(10, 10, 10)):
        x = self.setup(y=y, x0=x0, niter=niter, damp=damp, tol=tol, show=show)
        x = self.run(x, niter, show=show, itershow=itershow)
        self.finalize(show)
        return x, self.istop, self.iiter, self.r1norm, self.r2norm, self.cost


# ---- LSQR -----------------------------------------------------------------------------------------------------------
def _zeros_like(a):
    if isinstance(a, DistributedArray):
        return a.zeros_like()
    from ..StackedArray import StackedDistributedArray
    return StackedDistributedArray([_zeros_like(d) for d in a.distarrays], a.base_comm)


class LSQR(_DeviceLoopSolver):
    """LSQR (Paige & Saunders 1982) with pylops 2.x's ``LSQR`` interface: ``setup / step / run / finalize / solve``.
    An extension: pylops-mpi has no LSQR.  The iterates, stopping tests, ``istop`` (0-7) and the estimates are those
    of ``scipy.sparse.linalg.lsqr`` with ``iter_lim = niter`` and the same ``damp, atol, btol, conlim, calc_var, x0``.

    ONE fused iteration (``_body``) runs every mode: u and v stay unnormalised with their scales folded into the
    device coefficients of the next combination, the scalar recurrence runs on the device (``b2_lsqr_scalars``) and
    the model-side update is one pass (``b2_lsqr_update``).  ``run()`` replays the body as a CUDA graph in blocks
    and reads the scalar history once per block; a stop inside a block sets a device flag that turns the rest of
    the block into no-ops for x, w, var and the scalars.  ``step()`` runs the same body eagerly."""

    _BLOCK = 8

    def _print_step(self, x) -> None:
        x0 = (x if isinstance(x, DistributedArray) else x[0]).local_array.reshape(-1)[0].item()
        strx = f"{x0:1.2e}   " if isinstance(x0, complex) else f"{x0:11.4e}        "
        print(f"{self.iiter:6g}       " + strx + f"{self.r1norm:10.3e} {self.r2norm:10.3e}  {self.test1:8.1e} "
              f"{self.test2:8.1e} {self.anorm:8.1e} {self.acond:8.1e}")
        sys.stdout.flush()

    def setup(self, y, x0=None, damp: float = 0.0, atol: float = 1e-8, btol: float = 1e-8, conlim: float = 1e8,
              niter: int = 10, calc_var: bool = True, show: bool = False):
        self.y, self.damp, self.atol, self.btol, self.conlim = y, damp, atol, btol, conlim
        self.niter, self.calc_var = niter, calc_var
        self.ctol = 1 / conlim if conlim > 0 else 0.0
        ahu = None
        if x0 is None:
            self.U = y.copy()                               # scipy: u = b
            ahu = self.Op.rmatvec(self.U)                   # A^H u: v's direction and the model's layout
            x = _zeros_like(ahu)
        else:
            x = x0.copy()
            self.U = y - self.Op.matvec(x)
        self.rank = x.rank
        self._gen = _generic(x, self.U)
        if self._gen:
            bnorm, beta = float(y.norm().item()), float(self.U.norm().item())
        else:
            yy, uu = _self_dots([y, self.U]) if y.local_shape == self.U.local_shape else \
                (_self_dots([y])[0], _self_dots([self.U])[0])
            bnorm, beta = float(np.sqrt(yy)), float(np.sqrt(uu))
        if beta > 0:
            self.V = (1 / beta) * (self.Op.rmatvec(self.U) if ahu is None else ahu)
            alfa = float(self.V.norm().item()) if self._gen else float(np.sqrt(_self_dots([self.V])[0]))
        else:
            self.V, alfa = x.copy(), 0.0
        inv_alfa = 1 / alfa if alfa > 0 else 1.0
        self.W = inv_alfa * self.V                          # w = v
        self.var = _zeros_like(x)
        s = np.zeros(_NSTATE)
        s[[_ALFA, _BETA, _RHOBAR, _PHIBAR, _CS2, _INV_ALFA]] = alfa, beta, alfa, beta, -1.0, inv_alfa
        s[[_DAMP, _DAMPSQ, _ATOL, _BTOL, _CTOL, _BNORM, _ITER_LIM]] = damp, damp * damp, atol, btol, self.ctol, \
            bnorm, niter
        s[_CUB] = alfa * (1 / beta if beta > 0 else 1.0)
        self.iiter, self.istop = 0, 0
        self.r1norm = self.r2norm = beta
        self.anorm = self.acond = self.xnorm = 0.0
        self.arnorm = alfa * beta
        self.test1, self.test2 = 1.0, (alfa / beta if beta > 0 else 0.0)
        self._done = self.arnorm == 0                       # x0 solves the problem (scipy returns at once)
        s[_STOPPED] = float(self._done)
        self.cost: List = [self.r1norm]
        if self._gen:
            self._hs = s
        else:
            self._st = 2 if any(a._tdtype.is_complex for a in (x, self.U, self.V)) else 1
            self._dev = torch.from_numpy(s).to(x.local_array.device)
            self._hist = torch.zeros((max(niter, 1), _NHIST), dtype=torch.float64, device=self._dev.device)
            self._xs = x
        if show and self.rank == 0:
            self._print_solver(nbar=90)
            print(f"damp = {damp:20.14e}   calc_var = {calc_var:6g}")
            print(f"atol = {atol:8.2e}                 conlim = {conlim:8.2e}")
            print(f"btol = {btol:8.2e}                 niter = {niter:8g}")
            print("-" * 90 + "\n")
            print("    Itn          x[0]              r1norm     r2norm   Compatible   LS    Norm A   Cond A")
        return x

    # ---- fused path -------------------------------------------------------------------------------------------
    def _scalars(self, phase: int):
        _lib.check(_lib.lib.b2_lsqr_scalars(self._dev.data_ptr(), phase, self._hist.data_ptr(), self._hist.shape[0],
                                            _lib.stream()), "b2_lsqr_scalars")

    def _update(self, x):
        """x += t1 w, var += dk^2, w = inv_alfa v + t2 w and DD = |dk|^2 in one pass.  A BROADCAST model is updated
        whole on every rank, but DD is summed over this rank's share only (the re-scattered view of the
        reductions), so the all-reduce counts each element once."""
        from ..DistributedArray import Partition
        dev = self._dev
        ts = [a.local_array for a in (x, self.W, self.V)] + ([self.var.local_array] if self.calc_var else [])
        if any(not t.is_contiguous() for t in ts) or len({t.dtype for t in ts}) != 1:
            raise TypeError("lsqr: x, w, v and var must be contiguous and of one dtype")
        n = ts[0].numel()
        cuts = [0, n]
        if x.partition is not Partition.SCATTER and x.size > 1 and n:
            rows = ts[0].shape[0]
            ext = offsets(local_split_sizes(rows, x.size))
            cuts = [0, ext[x.rank] * (n // rows), ext[x.rank + 1] * (n // rows), n]
        own = 1 if len(cuts) == 4 else 0
        for k in range(len(cuts) - 1):
            a, b = cuts[k], cuts[k + 1]
            if b == a and k != own:
                continue
            p = [t.reshape(-1)[a:b] for t in ts]
            ptr = [t.data_ptr() if b > a else None for t in p]
            _lib.check(_lib.lib.b2_lsqr_update(_lib.ctx(), ptr[0], ptr[1], ptr[2], ptr[3] if self.calc_var else None,
                                               b - a, _lib.code(ts[0].dtype), dev.data_ptr() + 8 * _T1,
                                               dev.data_ptr() + 8 * _STOPPED,
                                               dev.data_ptr() + 8 * (_DD if k == own else _SCRATCH), _lib.stream()),
                       "b2_lsqr_update")

    def _body(self, x):
        """one LSQR iteration, no host synchronisation; its history row is written when the next body (or
        :meth:`_tail`) finishes it"""
        dev, st, sub = self._dev, self._st, x.sub_comm
        av = self.Op.matvec(self.V)
        if not _lincomb_dev_norm2(self.U, dev, _INV_ALFA, 1.0, av, dev, _CUB, -1.0, self.U, dev, _BB):
            _dots_device([self.U], dev, _BB)
        allreduce_(sub, dev[0:_DD + 1], "sum")             # BB and the previous iteration's DD
        self._scalars(0)
        ahu = self.Op.rmatvec(self.U)
        if not _lincomb_dev_norm2(self.V, dev, _CVA, 1.0, ahu, dev, _CVB, -1.0, self.V, dev, _AA):
            _dots_device([self.V], dev, _AA)
        allreduce_(sub, dev[_AA:_AA + st], "sum")
        self._scalars(1)
        self._update(x)

    def _tail(self, x, first: int):
        """finish the pending iteration and absorb the history rows from iteration ``first`` on (one host read)"""
        allreduce_(x.sub_comm, self._dev[_DD:_DD + 1], "sum")
        self._scalars(2)
        last = min(first + self._BLOCK, self._hist.shape[0])
        h = torch.cat((self._dev[_ITN:_ITN + 1], self._hist[first:last].reshape(-1))).cpu().numpy()
        itn = int(h[0])
        for row in h[1:].reshape(-1, _NHIST)[:itn - first]:
            self._absorb(row)

    def _absorb(self, row) -> None:
        (self.r1norm, self.r2norm, self.anorm, self.acond, self.arnorm, self.xnorm, self.test1, self.test2) = \
            (float(v) for v in row[:8])
        self.istop = int(row[8])
        self.iiter += 1
        self.cost.append(self.r1norm)

    def _ensure_rows(self, niter: int):
        if niter > self._hist.shape[0]:
            hist = torch.zeros((niter, _NHIST), dtype=torch.float64, device=self._hist.device)
            hist[:self._hist.shape[0]] = self._hist
            self._hist = hist

    # ---- generic path (stacked arrays): the same recurrence in DistributedArray operations -----------------------
    def _step_generic(self, x):
        s = self._hs
        if s[_STOPPED]:
            return x
        c = lambda i: float(s[i])                                   # noqa: E731  (NumPy scalars would broadcast)
        self.U = c(_INV_ALFA) * self.Op.matvec(self.V) - c(_CUB) * self.U
        s[_BB] = _absdot(self.U, self.U)
        lsqr_scalars_host(s, 0)
        self.V = c(_CVA) * self.Op.rmatvec(self.U) - c(_CVB) * self.V
        s[_AA] = _absdot(self.V, self.V)
        lsqr_scalars_host(s, 1)
        dk = c(_INV_RHO) * self.W
        x += c(_T1) * self.W
        if self.calc_var:
            self.var += dk * dk
        self.W = c(_INV_ALFA) * self.V + c(_T2) * self.W
        s[_DD] = _absdot(dk, dk)
        self._absorb(lsqr_scalars_host(s, 2))
        return x

    # ---- pylops interface --------------------------------------------------------------------------------------
    def step(self, x, show: bool = False):
        """one LSQR iteration: the fused body run eagerly, then its tests (one host synchronisation)"""
        if self._done or self.istop != 0:
            return x
        if self._gen:
            x = self._step_generic(x)
        else:
            self._ensure_rows(self.iiter + 1)
            self._body(x)
            self._tail(x, self.iiter)
        if show and self.rank == 0:
            self._print_step(x)
        return x

    def _run_blocks(self, x, niter: int):
        """the remaining iterations in blocks of :meth:`_iterate` (graph replays), one history read per block"""
        self._ensure_rows(niter)
        self._start_blocks()
        while self.iiter < niter and self.istop == 0:
            first = self.iiter
            for _ in range(min(self._BLOCK, niter - first)):
                self._iterate(x)
            self._tail(x, first)
        self._graph = None
        return x

    def run(self, x, niter: Optional[int] = None, show: bool = False, itershow=(10, 10, 10)):
        niter = self.niter if niter is None else niter
        if self._done:
            return x
        if not self._gen and not show and self._plain_callback() and niter - self.iiter > 0:
            return self._run_blocks(x, niter)
        while self.iiter < niter and self.istop == 0:
            showstep = bool(show and (self.iiter < itershow[0] or niter - self.iiter < itershow[1]
                                      or self.iiter % itershow[2] == 0))
            x = self.step(x, showstep)
            self.callback(x)
        return x

    def finalize(self, show: bool = False) -> None:
        self.tend = time.time()
        self.telapsed = self.tend - self.tstart
        self.cost = np.array(self.cost)
        if show and self.rank == 0:
            print(f"\nistop = {self.istop}   r1norm = {self.r1norm:8.1e}   anorm = {self.anorm:8.1e}   "
                  f"arnorm = {self.arnorm:8.1e}")
            print(f"itn   = {self.iiter}   r2norm = {self.r2norm:8.1e}   acond = {self.acond:8.1e}   "
                  f"xnorm  = {self.xnorm:8.1e}")
            self._print_finalize(nbar=90)

    def solve(self, y, x0=None, damp: float = 0.0, atol: float = 1e-8, btol: float = 1e-8, conlim: float = 1e8,
              niter: int = 10, calc_var: bool = True, show: bool = False, itershow=(10, 10, 10)):
        x = self.setup(y=y, x0=x0, damp=damp, atol=atol, btol=btol, conlim=conlim, niter=niter, calc_var=calc_var,
                       show=show)
        x = self.run(x, niter, show=show, itershow=itershow)
        self.finalize(show)
        return (x, self.istop, self.iiter, self.r1norm, self.r2norm, self.anorm, self.acond, self.arnorm, self.xnorm,
                self.var, self.cost)
