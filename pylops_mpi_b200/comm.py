"""Communicator shim: what the reference gets from ``mpi4py.MPI.Comm`` (host
metadata: ranks, sizes, tiny object collectives, ``Split``) plus the NCCL
communicator the device collectives run on (pylops_mpi/utils/_nccl.py:98-165).

One OS process per GPU (launched by ``torchrun``); host metadata travels over a
``torch.distributed`` gloo group, device buffers over NCCL through the C ABI
(``b2_comm_*``, ``b2_allreduce`` ...).  With a single process everything is
local and ``torch.distributed`` is never touched.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Any, List, Optional, Sequence

import numpy as np
import torch

__all__ = ["Comm", "COMM_WORLD", "get_comm_world", "SUM", "MAX", "MIN"]

SUM, MAX, MIN = "sum", "max", "min"


class Comm:
    """mpi4py-flavoured communicator over a torch.distributed (gloo) group.

    Mirrors the subset of ``MPI.Comm`` the reference uses on this path:
    ``Get_rank/Get_size/allgather/allreduce/bcast/Barrier/Split``
    (DistributedArray.py:67,99,453,536,899; BlockDiag.py:112-117; MatrixMult.py:305-306).
    """

    def __init__(self, rank: int = 0, size: int = 1, group=None, ranks: Optional[Sequence[int]] = None):
        self._rank = rank
        self._size = size
        self._group = group                     # torch.distributed group (None when size == 1)
        self._ranks = list(ranks) if ranks is not None else list(range(size))  # global ranks
        self._nccl = None                       # b2_comm handle (lazy)
        self._mailbox = None                    # b2_mailbox handle (lazy)
        self._mailbox_failed = False
        self._split_cache = {}

    # ---- mpi4py surface ------------------------------------------------------
    def Get_rank(self) -> int:
        return self._rank

    def Get_size(self) -> int:
        return self._size

    rank = property(Get_rank)
    size = property(Get_size)

    def allgather(self, obj: Any) -> List[Any]:
        if self._size == 1:
            return [obj]
        import torch.distributed as dist
        out = [None] * self._size
        dist.all_gather_object(out, obj, group=self._group)
        # torch orders group members by global rank; this communicator may not (Split keys)
        order = sorted(self._ranks)
        return [out[order.index(g)] for g in self._ranks]

    def allreduce(self, value, op: str = SUM):
        if self._size == 1:
            return value
        vals = self.allgather(value)
        if op == SUM:
            red = vals[0]
            for v in vals[1:]:
                red = red + v
            return red
        if op == MAX:
            return max(vals) if np.isscalar(vals[0]) else np.maximum.reduce(vals)
        if op == MIN:
            return min(vals) if np.isscalar(vals[0]) else np.minimum.reduce(vals)
        raise ValueError(f"unknown op {op}")

    def bcast(self, obj: Any, root: int = 0) -> Any:
        if self._size == 1:
            return obj
        import torch.distributed as dist
        box = [obj]
        dist.broadcast_object_list(box, src=self._ranks[root], group=self._group)
        return box[0]

    def Barrier(self):
        if self._size > 1:
            import torch.distributed as dist
            dist.barrier(group=self._group)

    barrier = Barrier

    def Split(self, color: int = 0, key: int = 0) -> "Comm":
        """MPI_Comm_split: collective over this communicator."""
        if self._size == 1:
            return Comm(0, 1)
        import torch.distributed as dist
        info = self.allgather((color, key, self._rank))
        mine = None
        for c in sorted({i[0] for i in info}):
            members = sorted([i for i in info if i[0] == c], key=lambda t: (t[1], t[2]))
            granks = [self._ranks[m[2]] for m in members]
            # every process of the parent must create every group, in the same order
            grp = dist.new_group(ranks=granks, backend="gloo") if len(granks) > 1 else None
            if c == color:
                my_idx = [m[2] for m in members].index(self._rank)
                mine = Comm(my_idx, len(granks), grp, granks)
        return mine

    # ---- NCCL side --------------------------------------------------------------
    @property
    def nccl(self):
        """b2_comm handle, created collectively on first use (size > 1 only)."""
        if self._size == 1:
            return None
        if self._nccl is None:
            from . import _lib
            uid = (C.c_char * 128)()
            if self._rank == 0:
                _lib.check(_lib.lib.b2_get_unique_id(uid), "b2_get_unique_id")
            raw = self.bcast(bytes(uid.raw), root=0)
            buf = (C.c_char * 128).from_buffer_copy(raw)
            h = C.c_void_p()
            _lib.check(_lib.lib.b2_comm_create(self._rank, self._size, buf,
                                               torch.cuda.current_device(), C.byref(h)),
                       "b2_comm_create")
            self._nccl = h
        return self._nccl

    def _symm_map(self, nbytes: int):
        """COLLECTIVE: every rank allocates ``nbytes`` of IPC-mappable device memory, exports its IPC handle, the
        handles are allgathered and every rank maps every peer's buffer.  Returns ``(ok, my_ptr, ptrs)`` with
        ``ptrs[r]`` = rank r's buffer as addressable from this process (``ptrs[rank] == my_ptr``).  A failed
        allocation or export on any rank fails every rank (the flag travels with the handles); ``ok`` only covers
        this rank's mapping of its peers, so callers finish with one allgather of ``ok`` to agree."""
        from . import _lib
        ok, ptr, mine = 1, C.c_void_p(), b""
        try:
            _lib.check(_lib.lib.b2_symm_alloc(max(int(nbytes), 16), C.byref(ptr)), "b2_symm_alloc")
            if self._size > 1:
                h = (C.c_char * 64)()
                _lib.check(_lib.lib.b2_ipc_get_handle(ptr, h), "b2_ipc_get_handle")
                mine = bytes(h.raw)
        except Exception:
            ok = 0
        handles = self.allgather((ok, mine))
        if not all(hh[0] for hh in handles):
            return 0, ptr.value, None
        ptrs = []
        try:
            for r, (_, raw) in enumerate(handles):
                if r == self._rank:
                    ptrs.append(ptr.value)
                else:
                    q = C.c_void_p()
                    _lib.check(_lib.lib.b2_ipc_open_handle((C.c_char * 64).from_buffer_copy(raw), C.byref(q)),
                               "b2_ipc_open_handle")
                    ptrs.append(q.value)
        except Exception:
            return 0, ptr.value, None
        return 1, ptr.value, ptrs

    def symm_alloc(self, nbytes: int):
        """COLLECTIVE: every rank allocates ``nbytes`` of IPC-mappable device memory and maps every peer's
        buffer; returns ``(my_ptr, ptrs)`` with ``ptrs[r]`` = rank r's buffer as addressable from this process
        (``ptrs[rank] == my_ptr``).  Used for the peer-memory arenas of the fused compute + collective kernels.
        Raises on every rank when the allocation or the mapping failed on any rank."""
        ok, ptr, ptrs = self._symm_map(nbytes)
        if min(self.allgather(ok)) == 0:
            from . import _lib
            raise _lib.B200Error(f"symm_alloc of {int(nbytes)} bytes: the allocation or the CUDA IPC mapping "
                                 f"failed on at least one rank")
        return ptr, ptrs

    HALO_CAP = 4 << 20      # bytes per (parity, side) slot of the halo region of a mailbox

    @property
    def mailbox(self):
        """b2_mailbox handle: this rank's box of IPC-mapped device memory and its mapping of every peer's box, for
        the one-shot scalar and vector all-reduces, the all-gather and the halo exchange inside the stencil kernels
        over NVLink peer memory.  Created collectively on first use; None for one rank, for more than 8 ranks, or
        when the allocation or the CUDA IPC mapping fails on any rank"""
        hit = self._mailbox
        if hit is not None:           # hot enqueue path: no lookups once the mailbox exists
            return hit
        if self._size == 1 or self._size > 8 or self._mailbox_failed:
            return None
        from . import _lib
        ok, _, ptrs = self._symm_map(_lib.lib.b2_mailbox_bytes(self.HALO_CAP))
        hnd = C.c_void_p()
        if ok:
            try:
                _lib.check(_lib.lib.b2_mailbox_create(self._rank, self._size, (C.c_void_p * self._size)(*ptrs),
                                                      self.HALO_CAP, C.byref(hnd)), "b2_mailbox_create")
            except Exception:
                ok = 0
        if min(self.allgather(ok)) == 1:      # every rank zeroed its box headers and mapped its peers
            self._mailbox = hnd
        else:
            self._mailbox_failed = True
        return self._mailbox

    halo = peer_vec = mailbox   # earlier names of the mailbox, which bench.py reads

    def split_by_mask(self, mask: Sequence[int]) -> "Comm":
        """cached ``Split(color=mask[rank], key=rank)`` (DistributedArray.py:74-100)"""
        key = tuple(int(m) for m in mask)
        sub = self._split_cache.get(key)
        if sub is None:
            sub = self._split_cache[key] = self.Split(color=key[self._rank], key=self._rank)
        return sub

    def __repr__(self):
        return f"<b200 Comm rank={self._rank} size={self._size}>"


_WORLD: Optional[Comm] = None


def get_comm_world() -> Comm:
    """The world communicator (mpi4py's ``MPI.COMM_WORLD``).

    Under ``torchrun`` (WORLD_SIZE > 1) initialises ``torch.distributed`` with the
    gloo backend for host metadata if the application has not done so, and binds
    this process to ``cuda:LOCAL_RANK``.
    """
    global _WORLD
    if _WORLD is not None:
        return _WORLD
    world = int(os.environ.get("WORLD_SIZE", "1"))
    import torch.distributed as dist
    if world > 1 or dist.is_initialized():
        if not dist.is_initialized():
            dist.init_process_group(backend="gloo")
        rank, size = dist.get_rank(), dist.get_world_size()
        if torch.cuda.is_available():
            torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)) % torch.cuda.device_count())
        grp = dist.new_group(ranks=list(range(size)), backend="gloo") if size > 1 else None
        _WORLD = Comm(rank, size, grp, list(range(size)))
    else:
        _WORLD = Comm(0, 1)
    return _WORLD


class _WorldProxy:
    """``COMM_WORLD`` resolved lazily so importing the package never touches
    torch.distributed."""

    def __getattr__(self, name):
        return getattr(get_comm_world(), name)

    def __repr__(self):
        return repr(get_comm_world())


COMM_WORLD = _WorldProxy()


def resolve(comm) -> Comm:
    """accept a Comm, the COMM_WORLD proxy or None"""
    if comm is None or isinstance(comm, _WorldProxy):
        return get_comm_world()
    return comm
