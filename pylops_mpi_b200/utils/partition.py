"""Integer partition bookkeeping (bit-exact with the reference) and the
exchange plans derived from it.  Pure host code: no CUDA, no communication.

Because ``local_split`` is a closed formula and user-supplied ``local_shapes``
are complete lists, every rank can compute every other rank's extents; the
reference re-derives them with host collectives on every temporary array
(DistributedArray.py:345-358, 523-539; utils/decorators.py:61-62), this
module computes them once.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np


def local_split_sizes(n: int, size: int) -> List[int]:
    """extents of the balanced split of ``n`` items over ``size`` ranks
    (DistributedArray.py:62-71: remainder goes to the low ranks)."""
    q, r = divmod(int(n), int(size))
    return [q + 1 if i < r else q for i in range(size)]


def offsets(sizes: Sequence[int]) -> List[int]:
    out = [0]
    for s in sizes:
        out.append(out[-1] + int(s))
    return out


def repartition_plan(src_sizes: Sequence[int], dst_sizes: Sequence[int], rank: int
                     ) -> Tuple[List[Tuple[int, int, int]], List[Tuple[int, int, int]]]:
    """Plan the move of a 1-D block-partitioned vector from ``src_sizes`` to
    ``dst_sizes`` (same total).  Returns (sends, recvs) for ``rank``:
    sends = [(peer, src_local_offset, count)], recvs = [(peer, dst_local_offset, count)],
    peers in increasing order; the self-overlap appears in both lists with peer == rank.

    Generalises the neighbour-only ghost-cell shuffle of utils/decorators.py:61-72
    (which raises when a deficit exceeds the neighbour's extent) to arbitrary
    interval overlaps.
    """
    if sum(src_sizes) != sum(dst_sizes):
        raise ValueError(f"repartition needs equal totals: {sum(src_sizes)} != {sum(dst_sizes)}")
    so, do = offsets(src_sizes), offsets(dst_sizes)
    sends, recvs = [], []
    a0, a1 = so[rank], so[rank + 1]
    for p in range(len(dst_sizes)):
        lo, hi = max(a0, do[p]), min(a1, do[p + 1])
        if hi > lo:
            sends.append((p, lo - a0, hi - lo))
    b0, b1 = do[rank], do[rank + 1]
    for p in range(len(src_sizes)):
        lo, hi = max(b0, so[p]), min(b1, so[p + 1])
        if hi > lo:
            recvs.append((p, lo - b0, hi - lo))
    return sends, recvs


def reshaped_ghost_cells(arr_sizes: Sequence[int], x_sizes: Sequence[int], rank: int):
    """The reference's neighbour-only plan (utils/decorators.py:61-72), kept for
    the strict-parity check: returns (cells_front, cells_back, start_index)."""
    dif = np.cumsum(np.asarray(arr_sizes) - np.asarray(x_sizes))
    cells_front = abs(min(0, int(dif[rank - 1])))
    cells_back = max(0, int(dif[rank]))
    index = max(0, int(dif[rank - 1]))
    return cells_front, cells_back, index


def halo_plan(row_sizes: Sequence[int], rank: int, need_lo: int, need_hi: int):
    """Rows exchanged with rank-1 / rank+1 for a stencil of reach (need_lo, need_hi)
    over an axis-0 row-block partition.  Returns dict with
      recv_lo / recv_hi : rows this rank receives from below / above,
      send_lo / send_hi : rows this rank sends to rank-1 (its first rows) / rank+1 (its last rows).
    Raises the reference's ValueError (DistributedArray.py:918-923, 935-940) when a
    neighbour owns fewer rows than the stencil needs.
    """
    size = len(row_sizes)
    offs = offsets(row_sizes)
    n_glob = offs[-1]

    def recv_counts(r):
        lo = min(need_lo, offs[r])
        hi = min(need_hi, n_glob - offs[r + 1])
        if row_sizes[r] == 0:
            return 0, 0
        return lo, hi

    lo, hi = recv_counts(rank)
    if lo and row_sizes[rank - 1] < lo:
        raise ValueError(f"Local Shape at rank={rank - 1} along axis=0 should be > {lo}: "
                         f"dim(0) {row_sizes[rank - 1]} < {lo}; to achieve this use "
                         f"NUM_PROCESSES <= {max(1, n_glob // lo)}")
    if hi and row_sizes[rank + 1] < hi:
        raise ValueError(f"Local Shape at rank={rank + 1} along axis=0 should be > {hi}: "
                         f"dim(0) {row_sizes[rank + 1]} < {hi}; to achieve this use "
                         f"NUM_PROCESSES <= {max(1, n_glob // hi)}")
    send_lo = recv_counts(rank - 1)[1] if rank > 0 else 0          # what rank-1 wants above it
    send_hi = recv_counts(rank + 1)[0] if rank < size - 1 else 0   # what rank+1 wants below it
    return {"recv_lo": lo, "recv_hi": hi, "send_lo": send_lo, "send_hi": send_hi}


def halo_launches(nloc: int, nl: int, nh: int, n_lo: int, n_hi: int):
    """Stencil launches of one rank's block of ``nloc`` rows, for a stencil of reach (nl, nh) and n_lo / n_hi
    received halo rows (``halo_plan``'s recv_lo / recv_hi).  Returns [(begin, end, lo, hi, after_exchange)] in
    launch order: local rows [begin, end) with ``lo`` halo rows below ``begin`` (the received rows when begin == 0,
    local rows otherwise) and ``hi`` rows from ``end`` on (the received rows when end == nloc).

    A block too short to overlap is one launch after the exchange.  Otherwise the interior rows go first, while
    the halo rows travel: they start at ``nl`` when rows are received below (not at ``n_lo``: a neighbour block
    next to a global edge can send fewer rows than the reach, and row n_lo still needs ``nl`` rows below it), and
    end at ``nloc - nh`` likewise; the one or two edge launches follow the exchange."""
    if nloc < 2 * (nl + nh) + 1:
        return [(0, nloc, n_lo, n_hi, True)]
    i0 = nl if n_lo else 0
    i1 = nloc - nh if n_hi else nloc
    out = [(i0, i1, min(nl, i0), min(nh, nloc - i1), False)]
    if i0:
        out.append((0, i0, n_lo, min(nh, nloc - i0), True))
    if i1 < nloc:
        out.append((i1, nloc, min(nl, i1), n_hi, True))
    return out
