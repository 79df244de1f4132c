"""``MPIFirstDerivative`` (pylops_mpi/basicoperators/FirstDerivative.py:18-319).

Per-rank apply = ONE stencil kernel launch (csrc/stencil.cu) on the rank's row
block plus one grouped NCCL exchange of <= 2 halo rows with rank +/- 1.  The
reference performs up to four separate ghost-cell exchanges and ~5 full-array
temporaries per call (:221-247, :276-319); here the adjoint is the exact
transpose stencil, generated from the forward taps, and needs the same single
exchange.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .. import _lib
from ..comm import COMM_WORLD
from ..Distributed import group, send, recv
from ..DistributedArray import DistributedArray, Partition
from ..LinearOperator import MPILinearOperator
from ..utils.decorators import reshaped
from ..utils.partition import halo_launches, halo_plan, offsets

_KINDS = {"forward": _lib.FD_FORWARD, "backward": _lib.FD_BACKWARD, "centered": _lib.FD_CENTERED}


class MPIFirstDerivative(MPILinearOperator):
    """First derivative along axis 0 of a ``dims``-shaped model distributed by
    row blocks.  Same constructor as the reference (FirstDerivative.py:84-91)."""

    def __init__(self, dims, sampling: float = 1.0, kind: str = "centered", edge: bool = False,
                 order: int = 3, base_comm=COMM_WORLD, dtype=np.float64):
        self.dims = tuple(int(d) for d in (dims if np.ndim(dims) else (dims,)))
        shape = (int(np.prod(self.dims)),) * 2
        super().__init__(shape=shape, dtype=np.dtype(dtype), base_comm=base_comm)
        self.sampling = sampling
        self.kind = kind
        self.edge = edge
        self.order = order
        self._register_multiplications(self.kind, self.order)
        self._plan_cache = {}

    def _register_multiplications(self, kind: str, order: int) -> None:
        # FirstDerivative.py:104-127 (same error behaviour)
        if kind == "forward" or kind == "backward":
            pass
        elif kind == "centered":
            if order not in (3, 5):
                raise NotImplementedError("'order' must be '3, or '5'")
        else:
            raise NotImplementedError("'kind' must be 'forward', 'centered', or 'backward'")
        self._kind_code = _KINDS[kind]

    # ---- hooks (MPISecondDerivative overrides these two) --------------------------------------------
    def _halo_need(self, adjoint: bool):
        need_lo, need_hi = C.c_int(), C.c_int()
        _lib.check(_lib.lib.b2_first_derivative_halo(self._kind_code, self.order, int(adjoint),
                                                     C.byref(need_lo), C.byref(need_hi)), "b2_first_derivative_halo")
        return need_lo.value, need_hi.value

    _deriv = 1      # MPISecondDerivative: 2 (same fused peer-halo entry point)

    def _kernel(self, ctx, xp, yp, lop, lo_n, hip, hi_n, nrows, ncols, row0, adjoint, code):
        _lib.check(_lib.lib.b2_first_derivative(ctx, xp, yp, lop, lo_n, hip, hi_n, nrows, ncols, row0, self.dims[0],
                                                self._kind_code, self.order, int(self.edge), float(self.sampling),
                                                adjoint, code, _lib.stream()), "b2_first_derivative")

    def _matvec(self, x: DistributedArray) -> DistributedArray:
        if x.partition is Partition.BROADCAST:
            x = DistributedArray.to_dist(x=x.local_array, base_comm=x.base_comm)
        return self._hmatvec(x)

    def _rmatvec(self, x: DistributedArray) -> DistributedArray:
        if x.partition is Partition.BROADCAST:
            x = DistributedArray.to_dist(x=x.local_array, base_comm=x.base_comm)
        return self._hrmatvec(x)

    @reshaped
    def _hmatvec(self, x: DistributedArray) -> DistributedArray:
        return self._apply(x, adjoint=False)

    @reshaped
    def _hrmatvec(self, x: DistributedArray) -> DistributedArray:
        return self._apply(x, adjoint=True)

    def _apply(self, x: DistributedArray, adjoint: bool) -> DistributedArray:
        xl = x.local_array
        tdt = xl.dtype
        # everything that depends only on (partition, dtype, direction) is pure integer work: once per key
        key = (tuple(x._local_shapes), tdt, bool(adjoint), x.mask is None, x.rank, x.size)
        cached = self._plan_cache.get(key)
        if cached is None:
            # complex data: the stencil has real taps -> treat as 2x wider real rows
            real_dt = {torch.complex64: torch.float32, torch.complex128: torch.float64}.get(tdt, tdt)
            if real_dt not in (torch.float32, torch.float64):
                raise TypeError(f"MPIFirstDerivative supports float32/64 and complex64/128, got {tdt}")
            mult = 2 if tdt.is_complex else 1
            rows = [s[0] for s in x._local_shapes]
            need_lo, need_hi = self._halo_need(adjoint)
            plan = halo_plan(rows, x.rank, need_lo, need_hi) if x.size > 1 else None
            ncols = int(np.prod(self.dims[1:])) * mult if len(self.dims) > 1 else mult
            esz = 4 if real_dt is torch.float32 else 8
            vec = 16 // esz
            # fused peer-halo path: the choice uses rank-invariant data only (global row split, dtype, ncols)
            peer_ok = (x.size > 1 and min(rows) >= max(need_lo, need_hi, 1) and ncols % vec == 0
                       and ncols // vec >= 8 and 2 * ncols * esz <= x.base_comm.HALO_CAP
                       and x.base_comm.size == x.size and x.mask is None)
            cached = self._plan_cache[key] = (rows, offsets(rows)[x.rank], need_lo, need_hi, plan, real_dt, ncols,
                                              _lib.code(real_dt), peer_ok, [tuple(s) for s in x._local_shapes],
                                              tuple(x.global_shape))
        rows, row0, nl, nh, plan, real_dt, ncols, code, peer_ok, lshapes, gshape = cached
        nloc = rows[x.rank]
        y = DistributedArray._internal(gshape, lshapes, x.base_comm, tdt, axis=x.axis)    # no mask, as :144-145
        if nloc == 0:
            return y
        yl = y.local_array
        if tdt.is_complex:
            xr, yr = torch.view_as_real(xl).reshape(nloc, ncols), torch.view_as_real(yl).reshape(nloc, ncols)
        else:
            xr, yr = xl.reshape(nloc, ncols), yl.reshape(nloc, ncols)
        ctx = _lib.ctx()

        def launch(r_begin, r_end, lo_t, lo_n, hi_t, hi_n):
            """stencil on local rows [r_begin, r_end) with explicit halo tensors"""
            if r_end <= r_begin:
                return
            self._kernel(ctx, xr[r_begin:].data_ptr(), yr[r_begin:].data_ptr(),
                         lo_t.data_ptr() if lo_n else None, lo_n, hi_t.data_ptr() if hi_n else None, hi_n,
                         r_end - r_begin, ncols, row0 + r_begin, int(adjoint), code)

        if x.size == 1:
            self._kernel(ctx, xr.data_ptr(), yr.data_ptr(), None, 0, None, 0, nloc, ncols, row0, int(adjoint), code)
            return y
        # fused path: halo rows are pushed / awaited INSIDE the stencil kernel over NVLink peer memory (ONE launch,
        # no NCCL, no side stream)
        if peer_ok:
            mailbox = x.base_comm.mailbox
            if mailbox is not None:
                if xr.data_ptr() % 16:        # never branch on a rank-local property: stage a mis-aligned view
                    xr = xr.clone()
                _lib.check(_lib.lib.b2_derivative_peer(ctx, mailbox, xr.data_ptr(), yr.data_ptr(), nloc, ncols,
                                                       row0, self.dims[0], self._deriv, self._kind_code, self.order,
                                                       int(self.edge), float(self.sampling), int(adjoint), code,
                                                       _lib.stream()), "b2_derivative_peer")
                return y
        n_lo, n_hi = plan["recv_lo"], plan["recv_hi"]
        lo = torch.empty((n_lo, ncols), dtype=real_dt, device=xl.device) if n_lo else None
        hi = torch.empty((n_hi, ncols), dtype=real_dt, device=xl.device) if n_hi else None

        def exchange():
            with group(x.base_comm):
                if plan["send_lo"]:
                    send(x.base_comm, xr[:plan["send_lo"]], x.rank - 1)
                if plan["send_hi"]:
                    send(x.base_comm, xr[nloc - plan["send_hi"]:], x.rank + 1)
                if n_lo:
                    recv(x.base_comm, lo, x.rank - 1)
                if n_hi:
                    recv(x.base_comm, hi, x.rank + 1)

        steps = halo_launches(nloc, nl, nh, n_lo, n_hi)

        def run(b, e, lo_n, hi_n, _after):
            launch(b, e, lo if b == 0 else xr[b - lo_n:], lo_n, hi if e == nloc else xr[e:], hi_n)

        if steps[0][4]:
            # tiny block: exchange, then one launch
            exchange()
            run(*steps[0])
            return y
        # overlap: halo rows travel over NVLink on a side stream while the interior rows (whose
        # stencil never leaves this rank) are differentiated; two 1-2 row edge launches follow
        main = torch.cuda.current_stream()
        side = _side_stream(xl.device)
        ready = torch.cuda.Event()
        ready.record(main)
        with torch.cuda.stream(side):
            side.wait_event(ready)
            exchange()
            arrived = torch.cuda.Event()
            arrived.record(side)
        run(*steps[0])
        main.wait_event(arrived)
        for s in steps[1:]:
            run(*s)
        return y


_SIDE = {}


def _side_stream(device):
    st = _SIDE.get(device)
    if st is None:
        st = _SIDE[device] = torch.cuda.Stream(device=device)
    return st
