"""Device collectives over NCCL/NVLink through the C ABI, and the
``DistributedMixIn`` dispatch surface of the reference
(pylops_mpi/Distributed.py:24-349).

All functions enqueue on the current torch CUDA stream and never synchronise
the host unless they must return host values.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .comm import Comm, resolve, SUM, MAX, MIN

_OPS = {SUM: _lib.SUM, MAX: _lib.MAX, MIN: _lib.MIN, None: _lib.SUM}
# one-shot peer-memory all-reduce below this payload, NCCL above (measured at 2 GPUs: 10.7 vs 11.1 us at
# 4 KB, 12.4 vs 13.9 us at 40 KB, 18.7 vs 14.9 us at 256 KB; NCCL needs ~34 us at 8 GPUs for <= 400 KB)
_PEER_VEC_MAX = min(int(_lib.lib.b2_peer_vec_max_bytes()), 64 * 1024)


def _flat(t: torch.Tensor) -> torch.Tensor:
    if not t.is_contiguous():
        raise ValueError("device collectives need contiguous tensors")
    return t


def allreduce_(comm: Comm, buf: torch.Tensor, op: str = SUM) -> torch.Tensor:
    """in-place Allreduce of a device tensor (utils/_nccl.py:203-240)"""
    if comm.size == 1 or buf.numel() == 0:
        return buf
    _flat(buf)
    if buf.dtype is torch.float64 and buf.numel() <= 8:
        # scalars (dot / norm / solver step lengths): one-shot all-reduce over NVLink peer memory
        mailbox = comm.mailbox
        if mailbox is not None:
            _lib.check(_lib.lib.b2_peer_allreduce(mailbox, buf.data_ptr(), buf.numel(), _OPS[op], _lib.stream()),
                       "b2_peer_allreduce")
            return buf
    if op in (SUM, None) and buf.dtype in (torch.float32, torch.float64) and \
            buf.numel() * buf.element_size() <= _PEER_VEC_MAX:
        # latency regime (e.g. MPIVStack adjoint with a small model): one-shot all-reduce over peer memory.
        # The transport is chosen from RANK-INVARIANT data only (dtype, element count, op): a rank-local
        # property such as pointer alignment could send ranks down different paths (and the lazy, collective
        # mailbox setup) and hang the job; a mis-aligned view is staged through an aligned scratch instead.
        # The mailbox keeps its sequence numbers in device memory: all calls on one communicator must be issued
        # on ONE stream (the current torch stream of the solver loop).
        mailbox = comm.mailbox
        if mailbox is not None:
            work = buf if buf.data_ptr() % 16 == 0 else buf.clone()
            _lib.check(_lib.lib.b2_peer_vec_allreduce(mailbox, work.data_ptr(), work.numel(), _lib.code(work.dtype),
                                                      _lib.stream()), "b2_peer_vec_allreduce")
            if work is not buf:
                buf.copy_(work)
            return buf
    _lib.check(_lib.lib.b2_allreduce(comm.nccl, buf.data_ptr(), buf.data_ptr(), buf.numel(),
                                     _lib.code(buf.dtype), _OPS[op], _lib.stream()), "b2_allreduce")
    return buf


_COUNTS_CACHE = {}      # counts tuple -> (ctypes size_t array, max count): hot enqueue path of the small gathers


def allgatherv(comm: Comm, send: torch.Tensor, counts: Sequence[int],
               out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """concatenation of every rank's flat ``send`` (counts[r] elements from rank r);
    replaces the pad-to-max allgather of utils/_nccl.py:363-403"""
    total = int(sum(counts))
    if out is None:
        out = torch.empty(total, dtype=send.dtype, device=send.device)
    if comm.size == 1:
        out.view(-1)[:total].copy_(send.reshape(-1))
        return out
    _flat(send)
    key = tuple(counts)
    hit = _COUNTS_CACHE.get(key)
    if hit is None:
        if len(_COUNTS_CACHE) > 256:
            _COUNTS_CACHE.clear()
        hit = _COUNTS_CACHE[key] = ((C.c_size_t * len(key))(*[int(c) for c in key]), max(int(c) for c in key))
    arr, cmax = hit
    if cmax * send.element_size() <= _PEER_VEC_MAX:
        # latency regime: one-shot all-gather over peer memory (rank-invariant choice: counts and dtype only)
        mailbox = comm.mailbox
        if mailbox is not None:
            _lib.check(_lib.lib.b2_peer_vec_allgatherv(mailbox, send.data_ptr() if send.numel() else None,
                                                       out.data_ptr(), arr, _lib.code(send.dtype), _lib.stream()),
                       "b2_peer_vec_allgatherv")
            return out
    _lib.check(_lib.lib.b2_allgatherv(comm.nccl, send.data_ptr(), out.data_ptr(), arr,
                                      _lib.code(send.dtype), _lib.stream()), "b2_allgatherv")
    return out


def bcast_(comm: Comm, buf: torch.Tensor, root: int = 0) -> torch.Tensor:
    if comm.size == 1 or buf.numel() == 0:
        return buf
    _flat(buf)
    _lib.check(_lib.lib.b2_bcast(comm.nccl, buf.data_ptr(), buf.numel(), _lib.code(buf.dtype),
                                 root, _lib.stream()), "b2_bcast")
    return buf


class group:
    """``with group():`` -> ncclGroupStart/End around p2p calls (utils/_nccl.py:357-360)"""

    def __init__(self, comm: Optional[Comm] = None):
        if comm is not None and comm.size > 1:
            comm.nccl  # create the communicator BEFORE opening the group

    def __enter__(self):
        _lib.check(_lib.lib.b2_group_start(), "b2_group_start")
        return self

    def __exit__(self, *exc):
        _lib.check(_lib.lib.b2_group_end(), "b2_group_end")
        return False


def send(comm: Comm, buf: torch.Tensor, dest: int):
    if buf.numel() == 0:
        return
    _flat(buf)
    _lib.check(_lib.lib.b2_send(comm.nccl, buf.data_ptr(), buf.numel(), _lib.code(buf.dtype), dest,
                                _lib.stream()), "b2_send")


def recv(comm: Comm, buf: torch.Tensor, source: int):
    if buf.numel() == 0:
        return buf
    _flat(buf)
    _lib.check(_lib.lib.b2_recv(comm.nccl, buf.data_ptr(), buf.numel(), _lib.code(buf.dtype), source,
                                _lib.stream()), "b2_recv")
    return buf


class DistributedMixIn:
    """Same method names / argument order as pylops_mpi/Distributed.py:35-349.
    ``base_comm_nccl`` is accepted for signature compatibility and ignored: the
    NCCL communicator lives inside ``base_comm`` (a :class:`Comm`).  Host
    objects (ints, tuples) go through the host group, device tensors through
    NCCL."""

    def _allreduce(self, base_comm, base_comm_nccl, send_buf, recv_buf=None, op=SUM, engine="b200"):
        comm = resolve(base_comm)
        if isinstance(send_buf, torch.Tensor) and send_buf.is_cuda:
            out = send_buf.clone() if recv_buf is None else recv_buf.copy_(send_buf)
            return allreduce_(comm, out.contiguous(), op)
        return comm.allreduce(send_buf, op)

    def _allreduce_subcomm(self, sub_comm, base_comm_nccl, send_buf, recv_buf=None, op=SUM, engine="b200"):
        return self._allreduce(sub_comm, None, send_buf, recv_buf, op, engine)

    def _allgather(self, base_comm, base_comm_nccl, send_buf, recv_buf=None, engine="b200") -> List:
        comm = resolve(base_comm)
        if isinstance(send_buf, torch.Tensor) and send_buf.is_cuda:
            shapes = comm.allgather(tuple(send_buf.shape))
            counts = [int(np.prod(s)) for s in shapes]
            flat = allgatherv(comm, send_buf.contiguous().view(-1), counts)
            out, off = [], 0
            for s, c in zip(shapes, counts):
                out.append(flat[off:off + c].view(s))
                off += c
            return out
        return comm.allgather(send_buf)

    def _allgather_subcomm(self, sub_comm, base_comm_nccl, send_buf, recv_buf=None, engine="b200"):
        return self._allgather(sub_comm, None, send_buf, recv_buf, engine)

    def _bcast(self, base_comm, base_comm_nccl, send_buf, root=0, engine="b200"):
        comm = resolve(base_comm)
        if isinstance(send_buf, torch.Tensor) and send_buf.is_cuda:
            return bcast_(comm, send_buf, root)
        return comm.bcast(send_buf, root)

    def _send(self, base_comm, base_comm_nccl, send_buf, dest, tag=0, engine="b200"):
        send(resolve(base_comm), send_buf.contiguous(), dest)

    def _recv(self, base_comm, base_comm_nccl, recv_buf=None, source=0, count=None, tag=0, engine="b200"):
        return recv(resolve(base_comm), recv_buf, source)

    def _sendrecv(self, base_comm, base_comm_nccl, sendbuf, dest, sendtag, recvbuf, source,
                  recvtag, engine="b200"):
        comm = resolve(base_comm)
        with group(comm):
            send(comm, sendbuf.contiguous(), dest)
            recv(comm, recvbuf, source)
        return recvbuf
