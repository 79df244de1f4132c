"""``MPIFredholm1`` (pylops_mpi/signalprocessing/Fredholm1.py:14-171): batched
(per frequency slice) dense product with the kernel ``G`` split over ranks along
the slice axis; BROADCAST model in, BROADCAST data out via an NCCL Allgather(v)
written straight into the output buffer."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .. import _lib
from ..comm import COMM_WORLD, resolve
from ..DistributedArray import DistributedArray, Partition
from ..LinearOperator import MPILinearOperator

# products per slice (nx * ny * nz) from which float32 / complex64 slices run on the tensor-core plan; smaller slices
# take the SIMT kernel
TC_MIN_PRODUCTS = 32768


class MPIFredholm1(MPILinearOperator):
    def __init__(self, G, nz: int = 1, saveGt: bool = False, usematmul: bool = True,
                 base_comm=COMM_WORLD, dtype="float64", fused=None, scatter_data: bool = False) -> None:
        base_comm = resolve(base_comm)
        # scatter_data=True (extension used by the frequency-domain MDC, waveeqprocessing/MDC.py): the DATA side stays
        # partitioned by slices -- forward takes the BROADCAST model and returns a SCATTER array holding only this rank's
        # slices (NO Allgather), the adjoint takes that SCATTER array and gathers the BROADCAST model.
        self._scatter_data = bool(scatter_data)
        self.nz = int(nz)
        if not isinstance(G, torch.Tensor):
            G = torch.as_tensor(np.asarray(G))
        self.nsl, self.nx, self.ny = (int(s) for s in G.shape)
        self.nsls = base_comm.allgather(self.nsl)
        if base_comm.Get_rank() == 0 and 1 in self.nsls:
            raise NotImplementedError(f'All ranks must have at least 2 or more '
                                      f'elements in the first dimension: '
                                      f'local split is instead {self.nsls}...')
        nslstot = int(sum(self.nsls))
        self.islstart = np.insert(np.cumsum(self.nsls)[:-1], 0, 0)
        self.islend = np.cumsum(self.nsls)
        self.dims = (nslstot, self.ny, self.nz)
        self.dimsd = (nslstot, self.nx, self.nz)
        shape = (int(np.prod(self.dimsd)), int(np.prod(self.dims)))
        super().__init__(shape=shape, dtype=np.dtype(dtype), base_comm=base_comm)
        _lib.ctx()
        self._tdtype = _lib.torch_dtype(dtype)
        self.G = G.to(device="cuda", dtype=self._tdtype).contiguous()
        # saveGt / usematmul change how the reference evaluates the adjoint (:147-167),
        # not its result; the batched kernel applies G^H on the fly.
        self.saveGt = saveGt
        self.usematmul = usematmul
        # fused=True: product + all-gather in ONE kernel over NVLink peer memory (IPC-mapped output
        # arenas); fused=False: product kernel, then one NCCL Allgatherv in place
        # fused=None (default): on when CUDA IPC peer mapping works between the ranks (probed by comm.mailbox)
        if fused is None:
            fused = base_comm.Get_size() > 1 and base_comm.mailbox is not None
        self._fused = bool(fused) and base_comm.Get_size() > 1 and not self._scatter_data
        if self._fused:
            esz = torch.empty(0, dtype=self._tdtype).element_size()
            self._arena = {}
            for adjoint in (False, True):
                nelem = nslstot * (self.ny if adjoint else self.nx) * self.nz
                for b in range(2):
                    self._arena[(adjoint, b)] = (*base_comm.symm_alloc(nelem * esz), nelem)
            self._toggle = {False: 0, True: 0}
            self._flag = torch.zeros(1, dtype=torch.float64, device="cuda")   # float64 -> peer-memory all-reduce
        # tensor-core plan (csrc/fredholm_tc.cu): float32 / complex64 products run on wgmma with fp16x2 split operands
        # (float32-class accuracy) for slices of >= TC_MIN_PRODUCTS products; G and G^H planes are built once here
        self._plan = None
        if self._tdtype in (torch.float32, torch.complex64) and \
                self.nx * self.ny * self.nz >= TC_MIN_PRODUCTS and self.nsl > 0:
            h = C.c_void_p()
            _lib.check(_lib.lib.b2_fredholm_plan_create(_lib.ctx(), self.G.data_ptr(), self.nsl, self.nx, self.ny, self.nz,
                                                        _lib.code(self._tdtype), C.byref(h)), "b2_fredholm_plan_create")
            self._plan = h

    def __del__(self):
        plan = getattr(self, "_plan", None)
        if plan is not None:
            try:
                _lib.lib.b2_fredholm_plan_destroy(plan)
            except Exception:
                pass
            self._plan = None

    def _product(self, x_ptr: int, y_ptr: int, adjoint: bool, peers=()):
        """this rank's slices: y = op(G) x on the tensor-core plan when one was built, the SIMT kernel otherwise.
        ``peers``: y's position in the other ranks' IPC-mapped arenas; the epilogue stores every output element
        there too (fused all-gather)"""
        arr = (C.c_void_p * len(peers))(*peers) if peers else None
        if self._plan is not None:
            _lib.check(_lib.lib.b2_fredholm_apply(self._plan, x_ptr, y_ptr, arr, len(peers), int(adjoint),
                                                  _lib.stream()), "b2_fredholm_apply")
        elif peers:
            _lib.check(_lib.lib.b2_batched_gemm_allgather(_lib.ctx(), self.G.data_ptr(), x_ptr, y_ptr, arr, len(peers),
                                                          self.nsl, self.nx, self.ny, self.nz, int(adjoint),
                                                          _lib.code(self._tdtype), _lib.stream()),
                       "b2_batched_gemm_allgather")
        else:
            _lib.check(_lib.lib.b2_batched_gemm(_lib.ctx(), self.G.data_ptr(), x_ptr, y_ptr, self.nsl, self.nx, self.ny,
                                                self.nz, int(adjoint), _lib.code(self._tdtype), _lib.stream()),
                       "b2_batched_gemm")

    def _product_gathered(self, xs: torch.Tensor, y: DistributedArray, adjoint: bool) -> DistributedArray:
        """this rank's slices of op(G) x straight into their place in the BROADCAST ``y``, then ONE NCCL Allgatherv
        in place on the current stream brings in the other ranks' slices"""
        rank, pout = self.rank, (self.ny if adjoint else self.nx) * self.nz
        yflat = y.local_array.view(-1)
        mine = yflat[self.islstart[rank] * pout: self.islend[rank] * pout]
        if self.nsl:
            self._product(xs.data_ptr(), mine.data_ptr(), adjoint)
        if y.size > 1:
            comm = y.base_comm
            counts = (C.c_size_t * comm.size)(*[int(n) * pout for n in self.nsls])
            offs = (C.c_size_t * comm.size)(*[int(o) * pout for o in self.islstart])
            _lib.check(_lib.lib.b2_allgatherv_at(comm.nccl, mine.data_ptr(), yflat.data_ptr(), counts, offs,
                                                 _lib.code(self._tdtype), _lib.stream()), "b2_allgatherv_at")
        return y

    # ---- fused product + all-gather over peer memory ------------------------------------------------
    def _apply_fused(self, x: DistributedArray, adjoint: bool) -> DistributedArray:
        from ..Distributed import allreduce_
        rank, comm = self.rank, x.base_comm
        nin, nout = (self.nx, self.ny) if adjoint else (self.ny, self.nx)
        xl = x.local_array if x.local_array.dtype == self._tdtype else x.local_array.to(self._tdtype)
        per, pout = nin * self.nz, nout * self.nz
        xs = xl.reshape(-1)[self.islstart[rank] * per: self.islend[rank] * per]
        b = self._toggle[adjoint]
        self._toggle[adjoint] = 1 - b
        base, peers, nelem = self._arena[(adjoint, b)]
        off = int(self.islstart[rank]) * pout * xl.element_size()
        self._product(xs.data_ptr(), base + off, adjoint, [peers[r] + off for r in range(comm.Get_size()) if r != rank])
        # stream-ordered cross-rank completion: when this tiny Allreduce finishes every rank's product
        # kernel (and its peer stores) has finished
        allreduce_(comm, self._flag, "sum")
        y = DistributedArray(global_shape=self.shape[1] if adjoint else self.shape[0], base_comm=comm,
                             partition=x.partition, dtype=self._tdtype)
        # copy out of the (double-buffered) arena: the caller owns an ordinary array, as in the reference
        _lib.check(_lib.lib.b2_lincomb(_lib.ctx(), y.local_array.data_ptr(), _lib.cpair(1.0), base, None, None, nelem,
                                       _lib.code(self._tdtype), 0, _lib.stream()), "b2_lincomb")
        return y

    def _apply_scatter(self, x: DistributedArray, adjoint: bool) -> DistributedArray:
        rank = self.rank
        if not adjoint:
            if x.partition not in [Partition.BROADCAST, Partition.UNSAFE_BROADCAST]:
                raise ValueError(f"x should have partition={Partition.BROADCAST},{Partition.UNSAFE_BROADCAST}"
                                 f"Got  {x.partition} instead...")
            per = self.ny * self.nz
            xl = x.local_array if x.local_array.dtype == self._tdtype else x.local_array.to(self._tdtype)
            xs = xl.reshape(-1)[self.islstart[rank] * per: self.islend[rank] * per]
            y = DistributedArray(global_shape=self.shape[0], base_comm=x.base_comm, partition=Partition.SCATTER,
                                 local_shapes=[(int(n) * self.nx * self.nz,) for n in self.nsls], dtype=self._tdtype)
            if self.nsl:
                self._product(xs.data_ptr(), y.local_array.data_ptr(), False)
            return y
        if x.partition is not Partition.SCATTER:
            raise ValueError(f"x should have partition={Partition.SCATTER} Got {x.partition} instead...")
        xl = x.local_array if x.local_array.dtype == self._tdtype else x.local_array.to(self._tdtype)
        if xl.numel() != self.nsl * self.nx * self.nz:
            raise ValueError("scattered data does not match this rank's slices")
        y = DistributedArray(global_shape=self.shape[1], base_comm=x.base_comm, partition=Partition.BROADCAST,
                             dtype=self._tdtype)
        return self._product_gathered(xl.reshape(-1), y, True)

    def _apply(self, x: DistributedArray, adjoint: bool) -> DistributedArray:
        if self._scatter_data:
            return self._apply_scatter(x, adjoint)
        if x.partition not in [Partition.BROADCAST, Partition.UNSAFE_BROADCAST]:
            raise ValueError(f"x should have partition={Partition.BROADCAST},{Partition.UNSAFE_BROADCAST}"
                             f"Got  {x.partition} instead...")
        if self._fused:
            return self._apply_fused(x, adjoint)
        if x.size == 1 and self._plan is not None and x.local_array.dtype == self._tdtype:
            # single rank, tensor-core plan: one library call (the 18.6 us apply is otherwise host-bound)
            n = self.shape[1] if adjoint else self.shape[0]
            y = DistributedArray._internal((n,), [(n,)], x.base_comm, self._tdtype, partition=x.partition)
            self._product(x._cont().data_ptr(), y.local_array.data_ptr(), adjoint)
            return y
        rank = self.rank
        per = (self.nx if adjoint else self.ny) * self.nz
        xl = x.local_array if x.local_array.dtype == self._tdtype else x.local_array.to(self._tdtype)
        xs = xl.reshape(-1)[self.islstart[rank] * per: self.islend[rank] * per]
        y = DistributedArray(global_shape=self.shape[1] if adjoint else self.shape[0],
                             base_comm=x.base_comm, partition=x.partition, dtype=self._tdtype)
        return self._product_gathered(xs, y, adjoint)

    def _matvec(self, x: DistributedArray) -> DistributedArray:
        return self._apply(x, False)

    def _rmatvec(self, x: DistributedArray) -> DistributedArray:
        return self._apply(x, True)
