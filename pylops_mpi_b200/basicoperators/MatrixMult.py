"""``MPIMatrixMult`` -- distributed dense matrix product, "block" and "summa"
variants (pylops_mpi/basicoperators/MatrixMult.py:24-874).

Per-rank tile products run in libb200lops: ``b2_gemv`` when the local block has
a single column (HBM-bound), ``b2_gemm_bf16`` (wgmma tensor cores) for bf16
tiles with many columns, ``b2_gemm`` (SIMT) for float32/float64/complex
tiles.  Row / column sub-communicators are NCCL groups created once at
construction; the SUMMA adjoint keeps the reference's semantics but sources
each A^H tile from a transposed-grid copy exchanged ONCE at construction
(``saveAt``-style), turning the per-apply point-to-point tile routing of
MatrixMult.py:742-763 into a plain column broadcast.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Tuple

import numpy as np
import torch

from .. import _lib
from ..comm import COMM_WORLD, resolve, SUM
from ..Distributed import DistributedMixIn, allreduce_, allgatherv, bcast_, group, send, recv
from ..DistributedArray import DistributedArray, Partition
from ..LinearOperator import MPILinearOperator

__all__ = ["active_grid_comm", "block_gather", "local_block_split", "MPIMatrixMult"]


def active_grid_comm(base_comm, N: int, M: int):
    """MatrixMult.py:24-76: the square sub-grid of ranks that own data."""
    base_comm = resolve(base_comm)
    rank = base_comm.Get_rank()
    size = base_comm.Get_size()
    p_prime = math.isqrt(size)
    row, col = divmod(rank, p_prime)
    active_dim = min(N, M, p_prime)
    is_active = (row < active_dim and col < active_dim)
    # Split is collective: inactive ranks take part with a different colour
    new_comm = base_comm.Split(color=0 if is_active else 1, key=rank)
    if not is_active:
        return None, rank, row, col, False
    p_prime_new = math.isqrt(new_comm.Get_size())
    new_rank = new_comm.Get_rank()
    new_row, new_col = divmod(new_rank, p_prime_new)
    return new_comm, new_rank, new_row, new_col, True


def local_block_split(global_shape: Tuple[int, int], rank: int, comm) -> Tuple[slice, slice]:
    """MatrixMult.py:79-125 (integer bookkeeping, bit-exact)."""
    size = resolve(comm).Get_size()
    p_prime = math.isqrt(size)
    if p_prime * p_prime != size:
        raise RuntimeError(f"Number of processes must be a square number, "
                           f"provided {size} instead...")
    if not (isinstance(rank, int) and 0 <= rank < size):
        raise ValueError(f"rank must be an integer in [0, {size}), got {rank!r}")
    pr, pc = divmod(rank, p_prime)
    orig_r, orig_c = global_shape
    new_r = math.ceil(orig_r / p_prime) * p_prime
    new_c = math.ceil(orig_c / p_prime) * p_prime
    blkr, blkc = new_r // p_prime, new_c // p_prime
    rs, cs = pr * blkr, pc * blkc
    re, ce = min(rs + blkr, orig_r), min(cs + blkc, orig_c)
    return slice(rs, re), slice(cs, ce)


def block_gather(x: DistributedArray, orig_shape: Tuple[int, int], comm):
    """MatrixMult.py:128-175: assemble the 2-D block-distributed matrix on every rank."""
    comm = resolve(comm)
    p_prime = math.isqrt(comm.Get_size())
    if p_prime * p_prime != comm.Get_size():
        raise RuntimeError(f"Communicator size must be a perfect square, got {comm.Get_size()!r}")
    all_blks = x._allgather(comm, None, x.local_array)
    nr, nc = orig_shape
    br, bc = math.ceil(nr / p_prime), math.ceil(nc / p_prime)
    Cm = torch.zeros((nr, nc), dtype=all_blks[0].dtype, device=all_blks[0].device)
    for rank in range(p_prime * p_prime):
        pr, pc = divmod(rank, p_prime)
        rs, cs = pr * br, pc * bc
        re, ce = min(rs + br, nr), min(cs + bc, nc)
        if all_blks[rank].numel() != 0:
            Cm[rs:re, cs:ce] = all_blks[rank].reshape(re - rs, ce - cs)
    return Cm


def _to_device(A, dtype) -> torch.Tensor:
    if not isinstance(A, torch.Tensor):
        A = torch.as_tensor(np.asarray(A))
    return A.to(device="cuda", dtype=_lib.torch_dtype(dtype)).contiguous()


def _xdtype(adt: torch.dtype) -> torch.dtype:
    """dtype of the vectors an operator with matrix dtype ``adt`` works on"""
    return torch.float32 if adt is torch.bfloat16 else adt


def _cast_bf16(X: torch.Tensor) -> torch.Tensor:
    """float32 (k x ncol, contiguous) -> bfloat16 through the library's cast kernel (no eager torch pass)"""
    if X.dtype is not torch.float32 or not X.is_contiguous():
        return X.to(torch.bfloat16)
    out = torch.empty(X.shape, dtype=torch.bfloat16, device=X.device)
    rows, cols = (X.shape[0], X.shape[1]) if X.dim() == 2 else (1, X.numel())
    dst = (C.c_void_p * 1)(out.data_ptr())
    _lib.check(_lib.lib.b2_cast_bf16_multi(_lib.ctx(), X.data_ptr(), cols, rows, cols, dst, 1, cols, _lib.stream()),
               "b2_cast_bf16_multi")
    return out


def tile_product(A: torch.Tensor, X: torch.Tensor, Y: torch.Tensor, op: int, accumulate: bool):
    """Y (+)= op(A) X on the device.  A: 2-D tile; X: (k, ncol); Y: (m, ncol) contiguous."""
    m_a, n_a = A.shape
    m, k = (m_a, n_a) if op == _lib.OP_N else (n_a, m_a)
    ncol = X.shape[1]
    if m == 0 or ncol == 0:
        return Y
    if k == 0:
        if not accumulate:
            Y.zero_()
        return Y
    ctx, st = _lib.ctx(), _lib.stream()
    if A.dtype is torch.bfloat16:
        if ncol == 1:
            if accumulate:
                tmp = torch.empty_like(Y)
                _lib.check(_lib.lib.b2_gemv(ctx, A.data_ptr(), n_a, m_a, n_a, X.data_ptr(), tmp.data_ptr(),
                                            op, _lib.BF16, _lib.F32, st), "b2_gemv")
                one = _lib.cpair(1.0)
                _lib.check(_lib.lib.b2_lincomb(ctx, Y.data_ptr(), one, tmp.data_ptr(), one, Y.data_ptr(),
                                               Y.numel(), _lib.F32, 0, st), "b2_lincomb")
            else:
                _lib.check(_lib.lib.b2_gemv(ctx, A.data_ptr(), n_a, m_a, n_a, X.data_ptr(), Y.data_ptr(),
                                            op, _lib.BF16, _lib.F32, st), "b2_gemv")
            return Y
        if n_a % 8 or ncol % 8 or A.data_ptr() % 16 or X.data_ptr() % 16:
            # tile extents the TMA descriptors cannot address (row pitch not a multiple of 16 bytes): rare ragged
            # case -> float32 SIMT product of the same bf16-rounded A (float32 accumulate, X not re-rounded)
            Xf = X if X.dtype is torch.float32 else X.float()
            _lib.check(_lib.lib.b2_gemm(ctx, A.float().contiguous().data_ptr(), n_a, Xf.data_ptr(), ncol, Y.data_ptr(), ncol,
                                        m, ncol, k, op, int(accumulate), _lib.F32, st), "b2_gemm")
            return Y
        Xb = X if X.dtype is torch.bfloat16 else _cast_bf16(X)
        _lib.check(_lib.lib.b2_gemm_bf16(ctx, A.data_ptr(), n_a, Xb.data_ptr(), ncol, Y.data_ptr(), ncol,
                                         m, ncol, k, op, int(accumulate), st), "b2_gemm_bf16")
        return Y
    if ncol == 1 and not accumulate:
        _lib.check(_lib.lib.b2_gemv(ctx, A.data_ptr(), n_a, m_a, n_a, X.data_ptr(), Y.data_ptr(), op,
                                    _lib.code(A.dtype), _lib.code(X.dtype), st), "b2_gemv")
        return Y
    _lib.check(_lib.lib.b2_gemm(ctx, A.data_ptr(), n_a, X.data_ptr(), ncol, Y.data_ptr(), ncol, m, ncol, k,
                                op, int(accumulate), _lib.code(A.dtype), st), "b2_gemm")
    return Y


class _MPIBlockMatrixMult(DistributedMixIn, MPILinearOperator):
    """1-D block variant (MatrixMult.py:178-428): A split in row blocks over the
    grid columns, X in column blocks over the grid rows."""

    def __init__(self, A, M: int, saveAt: bool = False, base_comm=COMM_WORLD, dtype="float64",
                 base_comm_nccl=None) -> None:
        base_comm = resolve(base_comm)
        rank, size = base_comm.Get_rank(), base_comm.Get_size()
        self._P_prime = math.isqrt(size)
        self._C = self._P_prime
        if self._P_prime * self._C != size:
            raise Exception(f"Number of processes must be a square number, provided {size} instead...")
        self._col_id = rank % self._P_prime
        self._row_id = rank // self._P_prime
        self.base_comm = base_comm
        self._row_comm = base_comm.Split(color=self._row_id, key=self._col_id)
        self._col_comm = base_comm.Split(color=self._col_id, key=self._row_id)
        self.A = _to_device(A, dtype)
        if saveAt:
            self.At = self.A.T.conj().contiguous()
        rows = self._row_comm.allgather(int(self.A.shape[0]))
        self._row_counts = rows
        self.N = int(sum(rows))
        self.K = int(self.A.shape[1])
        self.M = int(M)
        block_cols = int(math.ceil(self.M / self._P_prime))
        blk_rows = int(math.ceil(self.N / self._P_prime))
        self._row_start = self._col_id * blk_rows
        self._row_end = min(self.N, self._row_start + blk_rows)
        self._col_start = self._row_id * block_cols
        self._col_end = min(self.M, self._col_start + block_cols)
        self._local_ncols = max(0, self._col_end - self._col_start)
        self._rank_col_lens = base_comm.allgather(self._local_ncols)
        total_ncols = int(np.sum(self._rank_col_lens))
        self.dims = (self.K, total_ncols)
        self.dimsd = (self.N, total_ncols)
        shape = (int(np.prod(self.dimsd)), int(np.prod(self.dims)))
        MPILinearOperator.__init__(self, shape=shape, dtype=_lib.numpy_dtype(_xdtype(self.A.dtype)),
                                   base_comm=base_comm)

    def _matvec(self, x: DistributedArray) -> DistributedArray:
        if x.partition != Partition.SCATTER:
            raise ValueError(f"x should have partition={Partition.SCATTER} Got {x.partition} instead...")
        xdt = _xdtype(self.A.dtype)
        y = DistributedArray(global_shape=(self.N * self.dimsd[1]),
                             local_shapes=[(self.N * c) for c in self._rank_col_lens],
                             mask=x.mask, partition=Partition.SCATTER, dtype=xdt, base_comm=x.base_comm)
        nc = self._rank_col_lens[self.rank]
        X = x.local_array.to(xdt).reshape(self.dims[0], nc)
        Yloc = torch.empty((self.A.shape[0], nc), dtype=xdt, device=X.device)
        tile_product(self.A, X.contiguous(), Yloc, _lib.OP_N, False)
        # row-comm Allgather + vstack == concatenation of row blocks (MatrixMult.py:370-377)
        counts = [r * nc for r in self._row_counts]
        allgatherv(self._row_comm, Yloc.view(-1), counts, out=y.local_array)
        return y

    def _rmatvec(self, x: DistributedArray) -> DistributedArray:
        if x.partition != Partition.SCATTER:
            raise ValueError(f"x should have partition={Partition.SCATTER}. Got {x.partition} instead.")
        xdt = _xdtype(self.A.dtype)
        y = DistributedArray(global_shape=(self.K * self.dimsd[1]),
                             local_shapes=[self.K * c for c in self._rank_col_lens],
                             mask=x.mask, partition=Partition.SCATTER, dtype=xdt, base_comm=x.base_comm)
        nc = self._local_ncols
        X = x.local_array.to(xdt).reshape(self.N, nc)
        X_tile = X[self._row_start:self._row_end, :].contiguous()
        Yloc = y.local_array.view(self.K, nc)
        if hasattr(self, "At"):
            tile_product(self.At, X_tile, Yloc, _lib.OP_N, False)
        else:
            tile_product(self.A, X_tile, Yloc, _lib.OP_H, False)
        allreduce_(self._row_comm, y.local_array, SUM)     # MatrixMult.py:420-426
        return y


class _MPISummaMatrixMult(DistributedMixIn, MPILinearOperator):
    """2-D SUMMA (MatrixMult.py:431-767) on a Pr x Pc process grid.

    The reference supports square grids only (`:566-567`); with the default ``grid=None`` this class
    requires a square world and reproduces its tiling, padding (`:590-602`) and per-rank outputs exactly.
    ``grid=(Pr, Pc)`` generalises to rectangular grids (BASELINE config 4 asks for 2 x 4): K is cut into
    L = lcm(Pr, Pc) panels; an A tile owns L/Pc panel columns, an X tile L/Pr panel rows; round l
    broadcasts A panel l along the grid row and X panel l along the grid column.

    Pipelining: panel l+1 is broadcast on a side stream (double buffers) while the tile product of
    panel l runs on the compute stream.  The adjoint needs, on grid row i, the panels
    {A_{r,l} : r < Pr, l in X-tile i}; they are re-distributed ONCE at construction over the Pc ranks
    of that row (same bytes as the A tile itself), replacing the reference's per-apply point-to-point
    tile routing (`:742-763`) by row broadcasts.
    """

    def __init__(self, A, M: int, saveAt: bool = False, base_comm=COMM_WORLD, dtype="float64",
                 base_comm_nccl=None, grid=None, replicate: bool = False, stationary: bool = False) -> None:
        self._replicate = bool(replicate)
        self._stationary = bool(stationary)
        base_comm = resolve(base_comm)
        rank, size = base_comm.Get_rank(), base_comm.Get_size()
        if grid is None:
            self._P_prime = math.isqrt(size)
            if self._P_prime * self._P_prime != size:
                raise Exception(f"Number of processes must be a square number, provided {size} instead...")
            Pr = Pc = self._P_prime
        else:
            Pr, Pc = int(grid[0]), int(grid[1])
            if Pr * Pc != size:
                raise Exception(f"grid {Pr}x{Pc} does not match {size} processes")
            self._P_prime = Pr
        self._Pr, self._Pc = Pr, Pc
        self._L = Pr * Pc // math.gcd(Pr, Pc)
        L = self._L
        self._row_id, self._col_id = divmod(rank, Pc)
        self.base_comm = base_comm
        self._row_comm = base_comm.Split(color=self._row_id, key=self._col_id)
        self._col_comm = base_comm.Split(color=self._col_id, key=self._row_id)
        A = _to_device(A, dtype)
        self.N = int(self._col_comm.allreduce(int(A.shape[0])))
        self.K = int(self._row_comm.allreduce(int(A.shape[1])))
        self.M = int(M)
        self._N_padded = math.ceil(self.N / Pr) * Pr
        self._K_padded = math.ceil(self.K / L) * L
        self._M_padded = math.ceil(self.M / Pc) * Pc
        self._bn, self._bm = self._N_padded // Pr, self._M_padded // Pc
        self._w = self._K_padded // L                       # panel width
        self._pa, self._px = L // Pc, L // Pr               # panels per A tile / per X tile
        bkA = self._w * self._pa
        if A.shape[0] > self._bn or A.shape[1] > bkA:
            raise ValueError(f"local A tile {tuple(A.shape)} larger than the grid tile ({self._bn}, {bkA})")
        if A.shape[0] != self._bn or A.shape[1] != bkA:
            A = torch.nn.functional.pad(A, (0, bkA - A.shape[1], 0, self._bn - A.shape[0]))
        # panel-major storage: panel la = columns [la*w, (la+1)*w) of the tile, contiguous (bn x w)
        self._A_panels = [A[:, la * self._w:(la + 1) * self._w].contiguous() for la in range(self._pa)]
        self.A = A if self._pa > 1 else self._A_panels[0]
        self._At_panels = self._exchange_adjoint_panels()
        self.dims = (self.K, self.M)
        self.dimsd = (self.N, self.M)
        shape = (int(np.prod(self.dimsd)), int(np.prod(self.dims)))
        MPILinearOperator.__init__(self, shape=shape, dtype=_lib.numpy_dtype(_xdtype(A.dtype)),
                                   base_comm=base_comm)
        self._side = None
        # local shapes of the output tiles of every rank, forward [0] and adjoint [1]
        self._y_shapes = (self._tile_shapes(self._bn, self.N), self._tile_shapes(self._w * self._px, self.K))
        if self._replicate:
            self._build_replicas()
        if self._stationary:
            self._setup_stationary()
        # the function, not a bound method: a reference cycle would keep the tiles alive after the operator is dropped
        self._product = (_MPISummaMatrixMult._product_stationary if self._stationary else
                         _MPISummaMatrixMult._product_replicated if self._replicate else
                         _MPISummaMatrixMult._product_summa)

    # ---- stationary-A mode: A never moves; X / Y panels are all-gathered, partial products reduce-scattered -------
    def _setup_stationary(self):
        """SUMMA re-broadcasts the STATIC A panels on every apply (MatrixMult.py:663-670: 768 MiB received per rank
        per apply at 32768^2 / 2x4) -- A is operator state, X changes.  Stationary-A keeps ONE copy of A per GPU in
        the reference's 2-D tile layout and moves only the small operand and the partial results:
          forward  Y_ij = sum_j' A_ij' X_j'j :  (1) every X tile is cast to bf16 and pushed (P2P stores) into the
                   gathered-operand arena of the ranks whose A tile covers its K range, (2) ONE local tensor-core product
                   A_ij (bn x kA) . Xg (kA x M) whose epilogue stores column block c straight into rank (i, c)'s
                   staging slot j over NVLink (the reduce-scatter rides on the epilogue), (3) fold the Pc slots.
          adjoint  the same with A^H: gather Y along the grid row, one product per A panel, staging at rank (r, c).
        Two flag barriers per apply (peer-memory mailbox kernels); ~4x fewer NVLink bytes than broadcasting A at
        M = 4096 and no replication of A (cf. ``replicate=True``)."""
        comm = self.base_comm
        A0 = self._A_panels[0]
        if A0.dtype is not torch.bfloat16:
            raise NotImplementedError("stationary=True serves the bf16 -> fp32 tensor-core path")
        if comm.Get_size() > 8:
            raise NotImplementedError("stationary=True maps at most 8 peers")
        self._kA = self._w * self._pa
        if self._bm % 32 or self._w % 8 or self._bn % 8:
            raise NotImplementedError("stationary=True needs M/Pc % 32 == 0 and 8-aligned tile extents")
        if comm.Get_size() > 1 and comm.mailbox is None:
            raise NotImplementedError("stationary=True needs CUDA IPC peer access between the ranks")
        self._A_full = (torch.cat(self._A_panels, dim=1) if self._pa > 1 else self._A_panels[0]).contiguous()
        Mp = self._bm * self._Pc
        bkX = self._w * self._px
        self._st_Mp = Mp
        sizes = {"XG": self._kA * Mp * 2, "YG": self._bn * Mp * 2,
                 "SF": self._Pc * self._bn * self._bm * 4, "SA": self._Pr * bkX * self._bm * 4}
        self._st = {k: comm.symm_alloc(v) for k, v in sizes.items()}      # name -> (my_ptr, ptrs by world rank)
        self._st_flag = torch.zeros(1, dtype=torch.float64, device="cuda")
        self._st_keep = []
        comm.Barrier()

    def _st_barrier(self):
        """stream-ordered cross-rank barrier: completes when every rank's preceding kernels (and their peer stores)
        have completed"""
        allreduce_(self.base_comm, self._st_flag, SUM)

    def _product_stationary(self, x_block: torch.Tensor, Y: torch.Tensor, adjoint: bool):
        lib, ctx, st = _lib.lib, _lib.ctx(), _lib.stream()
        Pr, Pc, pa, px, w = self._Pr, self._Pc, self._pa, self._px, self._w
        bn, bm, Mp, kA = self._bn, self._bm, self._st_Mp, self._kA
        bkX = w * px
        i, j = self._row_id, self._col_id
        rank_of = lambda r, c: r * Pc + c          # noqa: E731

        def cast_to(src, rows, dst_ptrs):
            arr = (C.c_void_p * len(dst_ptrs))(*dst_ptrs)
            _lib.check(lib.b2_cast_bf16_multi(ctx, src.data_ptr(), bm, rows, bm, arr, len(dst_ptrs), Mp, st),
                       "b2_cast_bf16_multi")

        def gemm_seg(a_ptr, lda, b_ptr, seg_ptrs, m, k, op):
            arr = (C.c_void_p * len(seg_ptrs))(*seg_ptrs)
            _lib.check(lib.b2_gemm_bf16_seg(ctx, a_ptr, lda, b_ptr, Mp, arr, len(seg_ptrs), bm, bm, m, Mp, k, op, st),
                       "b2_gemm_bf16_seg")

        if not adjoint:
            XG, SF = self._st["XG"], self._st["SF"]
            for lx in range(px):                 # my X panels -> the ranks whose A tile owns that K range
                l = i * px + lx
                jc, la = l // pa, l % pa
                dsts = [XG[1][rank_of(r, jc)] + ((la * w) * Mp + j * bm) * 2 for r in range(Pr)]
                cast_to(x_block[lx * w:(lx + 1) * w], w, dsts)
            self._st_barrier()
            segs = [SF[1][rank_of(i, c)] + (j * bn * bm) * 4 for c in range(Pc)]
            gemm_seg(self._A_full.data_ptr(), kA, XG[0], segs, bn, kA, _lib.OP_N)
            self._st_barrier()
            slots, nslots, rows_blk = SF[0], Pc, bn
        else:
            YG, SA = self._st["YG"], self._st["SA"]
            dsts = [YG[1][rank_of(i, c)] + (j * bm) * 2 for c in range(Pc)]
            cast_to(x_block, bn, dsts)
            self._st_barrier()
            for la in range(pa):                 # one product per A panel: its rows land in X-tile row block r
                l = j * pa + la
                r, lx = l // px, l % px
                segs = [SA[1][rank_of(r, c)] + (i * bkX * bm + lx * w * bm) * 4 for c in range(Pc)]
                gemm_seg(self._A_full.data_ptr() + la * w * 2, kA, YG[0], segs, w, bn, _lib.OP_H)
            self._st_barrier()
            slots, nslots, rows_blk = SA[0], Pr, bkX
        _lib.check(lib.b2_sum_slots(ctx, slots, rows_blk * bm, nslots, bm, Y.data_ptr(), rows_blk, bm, st), "b2_sum_slots")

    # ---- replicated-panel mode (spend HBM, not NVLink) --------------------------------
    def _build_replicas(self):
        """A is operator STATE, X changes every apply -- yet SUMMA re-broadcasts the A panels on every
        apply (`:663-670`), which makes a 32768^2 bf16 product on 8 GPUs NVLink-bound.  With 180 GB of
        HBM per GPU each rank can keep, once, (i) its whole grid-row panel A[i-rows, :] (forward) and
        (ii) its X-tile's column panel A[:, k-range(i)] (adjoint).  An apply is then ONE allgather of
        the small operand along the grid column + ONE local tile product at full tensor-core rate.
        Same sums as SUMMA (different association) -> same result within rounding."""
        Pr, Pc = self._Pr, self._Pc
        bn, w = self._bn, self._w
        Kp, bkX = self._K_padded, self._w * self._px
        tile = torch.cat(self._A_panels, dim=1) if self._pa > 1 else self._A_panels[0]   # (bn, bkA)
        if Pc > 1:
            flat = allgatherv(self._row_comm, tile.reshape(-1), [tile.numel()] * Pc)
            self._A_row = torch.cat([flat[c * tile.numel():(c + 1) * tile.numel()].view(bn, -1) for c in range(Pc)],
                                    dim=1).contiguous()                                   # (bn, Kp)
        else:
            self._A_row = tile
        # column panel for the adjoint: rows of all Pr grid rows, columns k-range(row_id)
        if Pr > 1:
            blocks, outgoing = [None] * Pr, []
            with group(self._col_comm):
                for r in range(Pr):
                    blk = self._A_row[:, r * bkX:(r + 1) * bkX].contiguous()
                    if r == self._row_id:
                        blocks[r] = blk
                    else:
                        outgoing.append(blk)
                        send(self._col_comm, blk, r)
                        blocks[r] = torch.empty((bn, bkX), dtype=tile.dtype, device=tile.device)
                        recv(self._col_comm, blocks[r], r)
            torch.cuda.synchronize()      # construction time: send buffers may now be released
            del outgoing
            # blocks[r] (received from grid row r) == A[r-rows, k-range(me)]
            self._A_col = torch.cat(blocks, dim=0).contiguous()
        else:
            self._A_col = self._A_row[:, :bkX].contiguous() if bkX != Kp else self._A_row

    def _gather_col(self, blk: torch.Tensor) -> torch.Tensor:
        """stack the (rows x bm) tiles of this grid column: (Pr*rows x bm)"""
        if self._Pr == 1:
            return blk
        flat = allgatherv(self._col_comm, blk.reshape(-1), [blk.numel()] * self._Pr)
        return flat.view(self._Pr * blk.shape[0], blk.shape[1])

    def _product_replicated(self, x_block: torch.Tensor, Y: torch.Tensor, adjoint: bool):
        if self._A_row.dtype is torch.bfloat16 and self._bm > 1:
            x_block = _cast_bf16(x_block)                 # halves the allgather payload
        Xcol = self._gather_col(x_block)
        if adjoint:
            tile_product(self._A_col, Xcol, Y, _lib.OP_H, False)
        else:
            tile_product(self._A_row, Xcol, Y, _lib.OP_N, False)

    # ---- grid bookkeeping ------------------------------------------------------------------------
    def _extent(self, blk: int, full: int, idx: int, nblk: int) -> int:
        """true (unpadded) extent of block idx out of nblk blocks of padded size blk"""
        return max(0, min(full, (idx + 1) * blk) - idx * blk)

    def _adj_panel_src(self, i: int, p: int):
        """adjoint panel p of grid row i is A_{r,l}: returns (r, l, owner rank, owner local panel)"""
        r = p // self._px
        l = i * self._px + p % self._px
        return r, l, r * self._Pc + l // self._pa, l % self._pa

    def _exchange_adjoint_panels(self):
        """one-off re-distribution for the adjoint: rank (i, jc) keeps panels p with p // pa == jc"""
        Pr, Pc, L, pa = self._Pr, self._Pc, self._L, self._pa
        me = self.base_comm.Get_rank()
        mine = [None] * pa
        if self.base_comm.Get_size() == 1:
            return list(self._A_panels)
        sends, recvs = [], []
        for i in range(Pr):
            for p in range(L):
                r, l, src, la = self._adj_panel_src(i, p)
                dst = i * Pc + p // pa
                if src == me and dst == me:
                    mine[p % pa] = self._A_panels[la]
                elif src == me:
                    sends.append((dst, self._A_panels[la]))
                elif dst == me:
                    buf = torch.empty_like(self._A_panels[0])
                    mine[p % pa] = buf
                    recvs.append((src, buf))
        with group(self.base_comm):
            for dst, t in sends:
                send(self.base_comm, t, dst)
            for src, t in recvs:
                recv(self.base_comm, t, src)
        return mine

    def _tile_shapes(self, rows_blk: int, rows_full: int):
        """unpadded local shape of every rank's (rows_blk x bm) tile, as the 1-tuples ``DistributedArray._internal``
        takes"""
        return [(self._extent(rows_blk, rows_full, r // self._Pc, self._Pr) *
                 self._extent(self._bm, self.M, r % self._Pc, self._Pc),) for r in range(self.size)]

    def _padded_block(self, x: DistributedArray, rows_blk: int, rows_full: int, xdt):
        local_r = self._extent(rows_blk, rows_full, self._row_id, self._Pr)
        local_m = self._extent(self._bm, self.M, self._col_id, self._Pc)
        blk = x.local_array.to(xdt).reshape(local_r, local_m)
        if local_r != rows_blk or local_m != self._bm:
            blk = torch.nn.functional.pad(blk, (0, self._bm - local_m, 0, rows_blk - local_r))
        return blk.contiguous(), local_r, local_m

    def _pipeline(self, nrounds, fetch, compute):
        """run `compute(l, bufs)` for l < nrounds with `fetch(l)` (the broadcasts of round l, returns
        bufs) issued one round ahead on a side stream"""
        if self.base_comm.Get_size() == 1:
            for l in range(nrounds):
                compute(l, fetch(l))
            return
        main = torch.cuda.current_stream()
        if self._side is None:
            self._side = torch.cuda.Stream()
        side = self._side
        start = torch.cuda.Event()
        start.record(main)
        side.wait_event(start)
        done_compute = [None, None]          # compute events guarding buffer reuse (slot l % 2)
        pending = None
        for l in range(nrounds + 1):
            nxt = None
            if l < nrounds:
                with torch.cuda.stream(side):
                    if done_compute[l % 2] is not None:
                        side.wait_event(done_compute[l % 2])
                    bufs = fetch(l)
                    ev = torch.cuda.Event()
                    ev.record(side)
                nxt = (l, bufs, ev)
            if pending is not None:
                pl, pbufs, pev = pending
                main.wait_event(pev)
                compute(pl, pbufs)
                ce = torch.cuda.Event()
                ce.record(main)
                done_compute[pl % 2] = ce
            pending = nxt

    # ---- pipelined SUMMA ----------------------------------------------------------------------------------
    def _product_summa(self, x_block: torch.Tensor, Y: torch.Tensor, adjoint: bool):
        w, pa, px = self._w, self._pa, self._px
        a_tmp = [torch.empty_like(self._A_panels[0]) for _ in range(2)] if self.size > 1 else None
        if not adjoint:
            # forward: Y_ij = sum_l A_i,l X_l,j  (MatrixMult.py:612-674)
            x_tmp = [torch.empty((w, self._bm), dtype=x_block.dtype, device=x_block.device) for _ in range(2)] \
                if self.size > 1 else None

            def fetch(l):
                a_root, la = l // pa, l % pa
                x_root, lx = l // px, l % px
                xp = x_block[lx * w:(lx + 1) * w]
                if self.size == 1:
                    return self._A_panels[la], xp
                a_k = self._A_panels[la] if self._col_id == a_root else a_tmp[l % 2]
                x_k = xp if self._row_id == x_root else x_tmp[l % 2]
                bcast_(self._row_comm, a_k, root=a_root)
                bcast_(self._col_comm, x_k, root=x_root)
                return a_k, x_k

            def compute(l, bufs):
                tile_product(bufs[0], bufs[1], Y, _lib.OP_N, accumulate=(l > 0))
        else:
            # adjoint: Xadj_ij = sum_r sum_{l in tile i} (A_r,l)^H Y_r,j  (MatrixMult.py:676-767)
            x_tmp = [torch.empty_like(x_block) for _ in range(2)] if self.size > 1 else None
            state = {"r": -1, "buf": None}

            def fetch(p):
                a_root = p // pa
                r = p // px
                if self.size == 1:
                    return self._At_panels[p % pa], x_block
                a_k = self._At_panels[p % pa] if self._col_id == a_root else a_tmp[p % 2]
                bcast_(self._row_comm, a_k, root=a_root)
                if r != state["r"]:               # Y_r,j is shared by the px panels of round-group r
                    y_k = x_block if self._row_id == r else x_tmp[r % 2]
                    bcast_(self._col_comm, y_k, root=r)
                    state["r"], state["buf"] = r, y_k
                return a_k, state["buf"]

            def compute(p, bufs):
                # Y needs no zero fill: round group 0 (p < px) stores every row slice lx without accumulating
                lx = p % px
                tile_product(bufs[0], bufs[1], Y[lx * w:(lx + 1) * w], _lib.OP_H, accumulate=(p // px > 0))

        self._pipeline(self._L, fetch, compute)

    # ---- one apply frame for the three products ---------------------------------------------------------------
    def _apply(self, x: DistributedArray, adjoint: bool) -> DistributedArray:
        """the mode's product writes the padded (rows_out x bm) output tile ``Y``: a view of ``y`` when this rank's
        tile is not ragged, else scratch whose unpadded part is copied out once"""
        if x.partition != Partition.SCATTER:
            raise ValueError(f"x should have partition={Partition.SCATTER}. Got {x.partition} instead." if adjoint else
                             f"x should have partition={Partition.SCATTER} Got {x.partition} instead...")
        bkX = self._w * self._px
        rows_in, full_in, rows_out, full_out = (self._bn, self.N, bkX, self.K) if adjoint else \
            (bkX, self.K, self._bn, self.N)
        xdt = _xdtype(self.A.dtype)
        y = DistributedArray._internal((full_out * self.M,), self._y_shapes[adjoint], x.base_comm, xdt, mask=x.mask)
        x_block, _, local_m = self._padded_block(x, rows_in, full_in, xdt)
        local_out = self._extent(rows_out, full_out, self._row_id, self._Pr)
        direct = local_out == rows_out and local_m == self._bm
        Y = y.local_array.view(rows_out, self._bm) if direct else \
            torch.empty((rows_out, self._bm), dtype=xdt, device=x_block.device)
        self._product(self, x_block, Y, adjoint)
        if not direct:
            y.local_array.copy_(Y[:local_out, :local_m].reshape(-1))
        return y

    def _matvec(self, x: DistributedArray) -> DistributedArray:
        return self._apply(x, False)

    def _rmatvec(self, x: DistributedArray) -> DistributedArray:
        return self._apply(x, True)

def MPIMatrixMult(A, M: int, saveAt: bool = False, base_comm=COMM_WORLD, kind: str = "summa",
                  dtype="float64", base_comm_nccl=None, grid=None, replicate: bool = False, stationary: bool = False):
    """Factory with the reference's signature (MatrixMult.py:770-874); ``grid=(Pr, Pc)`` is the
    rectangular-grid extension of the SUMMA variant, ``replicate=True`` its replicated-panel mode
    (A row / column panels kept per rank, one small allgather + one local product per apply)."""
    if kind == "summa":
        return _MPISummaMatrixMult(A, M, saveAt, base_comm, dtype, base_comm_nccl, grid=grid, replicate=replicate,
                                   stationary=stationary)
    elif kind == "block":
        return _MPIBlockMatrixMult(A, M, saveAt, base_comm, dtype, base_comm_nccl)
    else:
        raise NotImplementedError("kind must be summa or block")
