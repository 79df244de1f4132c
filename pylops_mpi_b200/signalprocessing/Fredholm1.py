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
from ..DistributedArray import _BCAST, DistributedArray, Partition
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
        esz = self.G.element_size()
        if self._fused:
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
        # by direction (index: adjoint): byte offsets of this rank's slices in the input (the scattered data holds only
        # them) and in the output, the local shapes of a gathered output, and the element counts / offsets of every
        # rank's slices in it
        size, start = base_comm.Get_size(), int(self.islstart[base_comm.Get_rank()])
        self._x_off = [start * self.ny * self.nz * esz, 0 if self._scatter_data else start * self.nx * self.nz * esz]
        self._y_shapes = [[(n,)] * size for n in self.shape]
        self._y_off = [start * n * self.nz * esz for n in (self.nx, self.ny)]
        self._gatherv = [((C.c_size_t * size)(*[int(k) * n * self.nz for k in self.nsls]),
                          (C.c_size_t * size)(*[int(o) * n * self.nz for o in self.islstart])) for n in (self.nx, self.ny)]
        # how an apply delivers its output, chosen once; the function, not a bound method, so that no reference cycle
        # delays __del__
        self._output = (MPIFredholm1._out_scattered if self._scatter_data else
                        MPIFredholm1._out_fused if self._fused else MPIFredholm1._out_gathered)

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

    def _local_slices(self, x: DistributedArray, adjoint: bool):
        """this rank's slices of ``x`` in the operator dtype: ``(tensor holding them, address of the first)``; the
        caller keeps the tensor alive until the product is enqueued"""
        xl = x._cont()
        if xl.dtype != self._tdtype:
            xl = xl.to(self._tdtype)
        return xl, xl.data_ptr() + self._x_off[adjoint]

    def _out_gathered(self, x_ptr: int, x: DistributedArray, adjoint: bool) -> DistributedArray:
        """this rank's slices of op(G) x straight into their place in the BROADCAST ``y``, then ONE NCCL Allgatherv
        in place on the current stream brings in the other ranks' slices"""
        shapes = self._y_shapes[adjoint]
        y = DistributedArray._internal(shapes[0], shapes, x.base_comm, self._tdtype,
                                       partition=Partition.BROADCAST if x.partition is Partition.SCATTER else x.partition)
        base = y.local_array.data_ptr()
        if self.nsl:
            self._product(x_ptr, base + self._y_off[adjoint], adjoint)
        if self.size > 1:
            counts, offs = self._gatherv[adjoint]
            _lib.check(_lib.lib.b2_allgatherv_at(x.base_comm.nccl, base + self._y_off[adjoint], base, counts, offs,
                                                 _lib.code(self._tdtype), _lib.stream()), "b2_allgatherv_at")
        return y

    def _out_scattered(self, x_ptr: int, x: DistributedArray, adjoint: bool) -> DistributedArray:
        """scatter_data: the forward output holds only this rank's slices (no gather); the adjoint gathers"""
        if adjoint:
            return self._out_gathered(x_ptr, x, True)
        y = DistributedArray._internal((self.shape[0],), [(int(n) * self.nx * self.nz,) for n in self.nsls],
                                       x.base_comm, self._tdtype)
        if self.nsl:
            self._product(x_ptr, y.local_array.data_ptr(), False)
        return y

    def _out_fused(self, x_ptr: int, x: DistributedArray, adjoint: bool) -> DistributedArray:
        """product and all-gather in one kernel over peer memory"""
        from ..Distributed import allreduce_
        rank, comm = self.rank, x.base_comm
        b = self._toggle[adjoint]
        self._toggle[adjoint] = 1 - b
        base, peers, nelem = self._arena[(adjoint, b)]
        off = self._y_off[adjoint]
        self._product(x_ptr, base + off, adjoint, [peers[r] + off for r in range(comm.Get_size()) if r != rank])
        # stream-ordered cross-rank completion: when this tiny Allreduce finishes every rank's product
        # kernel (and its peer stores) has finished
        allreduce_(comm, self._flag, "sum")
        shapes = self._y_shapes[adjoint]
        y = DistributedArray._internal(shapes[0], shapes, comm, self._tdtype, partition=x.partition)
        # copy out of the (double-buffered) arena: the caller owns an ordinary array, as in the reference
        _lib.check(_lib.lib.b2_lincomb(_lib.ctx(), y.local_array.data_ptr(), _lib.cpair(1.0), base, None, None, nelem,
                                       _lib.code(self._tdtype), 0, _lib.stream()), "b2_lincomb")
        return y

    def _apply(self, x: DistributedArray, adjoint: bool) -> DistributedArray:
        if self._scatter_data and adjoint:
            if x.partition is not Partition.SCATTER:
                raise ValueError(f"x should have partition={Partition.SCATTER} Got {x.partition} instead...")
            if x.local_array.numel() != self.nsl * self.nx * self.nz:
                raise ValueError("scattered data does not match this rank's slices")
        elif x.partition not in _BCAST:
            raise ValueError(f"x should have partition={Partition.BROADCAST},{Partition.UNSAFE_BROADCAST}"
                             f"Got  {x.partition} instead...")
        xl, x_ptr = self._local_slices(x, adjoint)      # xl holds the slices until the product is enqueued
        return self._output(self, x_ptr, x, adjoint)

    def _matvec(self, x: DistributedArray) -> DistributedArray:
        return self._apply(x, False)

    def _rmatvec(self, x: DistributedArray) -> DistributedArray:
        return self._apply(x, True)
