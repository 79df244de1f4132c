"""Multi-rank parity worker: run under torchrun with one process per GPU.  Every
check compares the GPU path at world size P with the CPU oracle simulating the
reference at the same P (per-rank outputs, not just gathered ones)."""
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import pylops_mpi_oracle as o  # noqa: E402
import pylops_mpi_b200 as pm  # noqa: E402

comm = pm.get_comm_world()
rank, P = comm.Get_rank(), comm.Get_size()


def host(t):
    return t.cpu().numpy()


def check(name, got, ref, rtol=1e-12, atol=1e-12):
    np.testing.assert_allclose(got, ref, rtol=rtol, atol=atol, err_msg=f"[rank {rank}] {name}")


# ---- DistributedArray ---------------------------------------------------------------------
np.random.seed(42)
for shape, axis in [((50, 51), 1), ((51, 50), 0), ((20, 21, 11), 1), ((600,), 0)]:
    a = np.random.normal(100, 100, shape)
    b = np.random.normal(300, 300, shape)
    A = pm.DistributedArray.to_dist(a, axis=axis)
    B = pm.DistributedArray.to_dist(b, axis=axis)
    assert A.local_shape == o.local_split(shape, P, rank, o.SCATTER, axis)
    assert A.local_shapes == o.local_shapes(shape, P, o.SCATTER, axis)
    check("asarray", host(A.asarray()), a, 0, 0)
    check("add", host((A + B).asarray()), a + b)
    al, bl = o.to_dist(a, P, axis=axis), o.to_dist(b, P, axis=axis)
    check("local", host(A.local_array), al[rank], 0, 0)
    check("dot", A.dot(B)[0], o.dot(al, bl)[rank], 1e-13, 0)
    for ord_ in (None, 1, np.inf, -np.inf, 0, 3):
        check(f"norm{ord_}", A.norm(ord_)[0], o.norm(al, ord_)[rank], 1e-13, 0)
    Bc = pm.DistributedArray.to_dist(a, partition=pm.Partition.BROADCAST)
    check("bcast dot", Bc.dot(Bc)[0], np.dot(a.ravel(), a.ravel()), 1e-13, 0)
    if len(shape) == 2:
        R = A.redistribute(1 - axis)
        check("redistribute", host(R.asarray()), a, 0, 0)
        assert R.local_shape == o.local_split(shape, P, rank, o.SCATTER, 1 - axis)
# masked sub-communicators (test_distributedarray.py:270-361)
if P >= 2:
    mask = [r % 2 for r in range(P)]
    x = np.arange(24.0 * P)
    X = pm.DistributedArray.to_dist(x, mask=mask)
    xl = o.to_dist(x, P)
    check("masked dot", X.dot(X)[0], o.dot(xl, xl, mask=mask)[rank], 1e-14, 0)
    check("masked norm", X.norm(1)[0], o.norm(xl, 1, mask=mask)[rank], 1e-14, 0)
# ghost cells
G = pm.DistributedArray.to_dist(np.arange(40.0 * P).reshape(10 * P, 4))
g = host(G.add_ghost_cells(cells_front=2, cells_back=1))
ref = o.add_ghost_cells(o.to_dist(np.arange(40.0 * P).reshape(10 * P, 4), P), 0, [2] * P, [1] * P)[rank]
check("ghost", g, ref, 0, 0)

# ---- array all-reduce: peer-memory one-shot path (small) and NCCL path (large) vs the exact sum --------
from pylops_mpi_b200.Distributed import allreduce_  # noqa: E402
for dt in (torch.float32, torch.float64):
    for nel in (1, 5, 9, 1000, 32768, 65536 if dt is torch.float32 else 32768, 70001, 300000):
        gen = torch.Generator(device="cuda").manual_seed(1234 + rank)
        v = torch.randint(-1000, 1000, (nel,), device="cuda", generator=gen).to(dt)     # integers: exact sums
        ref = torch.zeros(nel, dtype=dt, device="cuda")
        for r in range(P):
            g2 = torch.Generator(device="cuda").manual_seed(1234 + r)
            ref += torch.randint(-1000, 1000, (nel,), device="cuda", generator=g2).to(dt)
        for _ in range(3):                                                              # repeated: parity buffers
            w = v.clone()
            allreduce_(comm, w)
            assert torch.equal(w, ref), f"[rank {rank}] allreduce {dt} n={nel}"

# ---- MPIFirstDerivative (config 1 at P = world size, plus the test_derivative grid) ---------------
x = np.zeros((11, 21))
x[5, 10] = 1.0
Fop = pm.MPIFirstDerivative((11, 21))
try:
    refl = o.first_derivative(o.to_dist(x.ravel(), P), (11, 21))
    y = Fop @ pm.DistributedArray.to_dist(x.ravel())
    assert np.array_equal(host(y.local_array), refl[rank]), "config-1 KAT per-rank"
except ValueError:
    # the reference cannot run this split (SURVEY 8a: P=8); the native re-partition can
    y = Fop @ pm.DistributedArray.to_dist(x.ravel())
    e = np.zeros((11, 21))
    e[4, 10], e[6, 10] = 0.5, -0.5
    assert np.array_equal(host(y.asarray()), e.ravel())
rng = np.random.default_rng(42)
for dims, h in [((600,), 1.0), ((100, 151), 1.0), ((101, 51, 10), 0.4), ((79, 11, 5), 0.4), ((64 * P, 256), 1.0)]:
    for kind, order in [("forward", 3), ("backward", 3), ("centered", 3), ("centered", 5)]:
        for edge in (False, True):
            for dtype in (np.float64, np.complex128):
                n = int(np.prod(dims))
                xg = rng.normal(0, 10, n).astype(dtype)
                if dtype is np.complex128:
                    xg = xg + 1j * rng.normal(0, 10, n)
                xg = comm.bcast(xg, 0)
                Fop = pm.MPIFirstDerivative(dims, sampling=h, kind=kind, edge=edge, order=order, dtype=dtype)
                D = o.first_derivative_dense(dims[0], h, kind, edge, order)
                X = xg.reshape(dims[0], -1)
                for part in (pm.Partition.SCATTER, pm.Partition.BROADCAST):
                    xd = pm.DistributedArray.to_dist(xg, partition=part)
                    y, ya = Fop @ xd, Fop.H @ xd
                    check(f"fd {dims} {kind}{order} {edge}", host(y.asarray()), (D @ X).ravel())
                    check(f"fdH {dims} {kind}{order} {edge}", host(ya.asarray()), (D.T @ X).ravel())
                try:
                    refl = o.first_derivative(o.to_dist(xg, P), dims, h, kind, edge, order, False, dtype=dtype)
                    check("fd per-rank", host((Fop @ pm.DistributedArray.to_dist(xg)).local_array), refl[rank])
                except (ValueError, IndexError):
                    pass
                u = pm.DistributedArray.to_dist(comm.bcast(rng.normal(0, 10, n), 0).astype(dtype))
                v = pm.DistributedArray.to_dist(comm.bcast(rng.normal(0, 10, n), 0).astype(dtype))
                assert pm.dottest(Fop, u, v)

# ---- "next" rows: MPISecondDerivative (per-rank vs oracle) and MPILaplacian (vs dense) --------------------
for dims, h in [((600,), 1.0), ((100, 37), 0.4), ((41, 9, 6), 0.4)]:
    for kind in ("forward", "backward", "centered"):
        for edge in (False, True):
            n = int(np.prod(dims))
            xg = comm.bcast(rng.normal(0, 10, n), 0)
            Sop = pm.MPISecondDerivative(dims, sampling=h, kind=kind, edge=edge)
            D2 = o.second_derivative_dense(dims[0], h, kind, edge)
            X = xg.reshape(dims[0], -1)
            xd = pm.DistributedArray.to_dist(xg)
            check(f"sd {dims} {kind} {edge}", host((Sop @ xd).asarray()), (D2 @ X).ravel(), 1e-12, 1e-10)
            check(f"sdH {dims} {kind} {edge}", host((Sop.H @ xd).asarray()), (D2.T @ X).ravel(), 1e-12, 1e-10)
            try:
                refl = o.second_derivative(o.to_dist(xg, P), dims, h, kind, edge, False)
                check("sd per-rank", host((Sop @ xd).local_array), refl[rank], 1e-12, 1e-10)
            except (ValueError, IndexError):
                pass
    if len(dims) > 1:
        axes = tuple(range(len(dims)))
        Lop = pm.MPILaplacian(dims, axes=axes, weights=(1.0,) * len(axes), sampling=(1.0, 0.5, 2.0)[:len(axes)], edge=True)
        xg = comm.bcast(rng.normal(0, 10, int(np.prod(dims))), 0)
        ref = sum(o.derivative_along_axis(xg.reshape(dims), ax, o.second_derivative_dense(dims[ax], s, "centered", True))
                  for ax, s in zip(axes, (1.0, 0.5, 2.0)))
        check(f"laplacian {dims}", host((Lop @ pm.DistributedArray.to_dist(xg)).asarray()), ref.ravel(), 1e-11, 1e-9)

# ---- uneven row splits: 1-row blocks next to a global edge, applied on the split as given ---------------------
# (_apply directly: the public matvec re-partitions to the balanced split first).  A neighbour next to a global
# edge then sends fewer halo rows than the stencil's reach, and the overlapped exchange must still give every
# launch the rows it reads.
from pylops_mpi_b200.utils.partition import local_split_sizes  # noqa: E402
N = 12 * P
dims = (N, 5)
uneven = [[N]] if P == 1 else [[1] + local_split_sizes(N - 1, P - 1), local_split_sizes(N - 1, P - 1) + [1]]
if P >= 3:
    uneven.append([1] + local_split_sizes(N - 2, P - 2) + [1])
X = comm.bcast(rng.normal(0, 10, dims), 0)
ops = [(pm.MPIFirstDerivative(dims, kind="centered", edge=e, order=order),
        o.first_derivative_dense(N, 1.0, "centered", e, order), f"fd centered{order} edge={e}")
       for order in (3, 5) for e in (False, True)]
ops += [(pm.MPISecondDerivative(dims, kind=kind, edge=e), o.second_derivative_dense(N, 1.0, kind, e),
         f"sd {kind} edge={e}") for kind in ("forward", "backward", "centered") for e in (False, True)]
for rows in uneven:
    off = np.cumsum([0] + rows)
    xd = pm.DistributedArray(global_shape=dims, local_shapes=[(r, dims[1]) for r in rows], dtype=np.float64)
    xd[:] = X[off[rank]:off[rank + 1]]
    for Op, D, name in ops:
        for adjoint in (False, True):
            y = Op._apply(xd, adjoint=adjoint)
            ref = ((D.T if adjoint else D) @ X)[off[rank]:off[rank + 1]]
            check(f"{name} adj={adjoint} split={rows}", host(y.local_array), ref, 1e-12, 1e-10)

# ---- BlockDiag / VStack / HStack (test_blockdiag.py:24-71, test_stack.py:29-79) ---------------------
for ny, nx in [(101, 101), (301, 101)]:
    for dtype in (np.float64, np.complex128):
        blocks = [[((r + 1) * np.ones((ny, nx))).astype(dtype)] for r in range(P)]
        BD = pm.MPIBlockDiag([pm.MatrixMult(blocks[rank][0])])
        assert BD.shape == (P * ny, P * nx)
        xd = pm.DistributedArray(global_shape=P * nx, dtype=dtype)
        xd[:] = 1.0
        y = BD @ xd
        check("bd", host(y.local_array), (rank + 1) * nx * np.ones(ny), 1e-13, 0)
        yd = pm.DistributedArray(global_shape=P * ny, dtype=dtype)
        yd[:] = 1.0
        check("bdH", host((BD.H @ yd).local_array), (rank + 1) * ny * np.ones(nx), 1e-13, 0)
        assert pm.dottest(BD, xd, yd)
        VS = pm.MPIVStack([pm.MatrixMult(blocks[rank][0])])
        xb = pm.DistributedArray(global_shape=nx, partition=pm.Partition.BROADCAST, dtype=dtype)
        xb[:] = 1.0
        check("vs", host((VS @ xb).local_array), (rank + 1) * nx * np.ones(ny), 1e-13, 0)
        xr = VS.H @ yd
        assert xr.partition is pm.Partition.BROADCAST
        check("vsH", host(xr.local_array), sum(r + 1 for r in range(P)) * ny * np.ones(nx), 1e-13, 0)
        # random blocks + un-aligned flat input (re-partition path) vs oracle
        rb = [[comm.bcast(np.random.default_rng(7 + r).standard_normal((ny - r, nx)).astype(dtype), 0)] for r in range(P)]
        BD2 = pm.MPIBlockDiag([pm.MatrixMult(rb[rank][0])])
        xv = comm.bcast(np.random.default_rng(1).standard_normal(P * nx).astype(dtype), 0)
        check("bd2", host((BD2 @ pm.DistributedArray.to_dist(xv)).local_array), o.blockdiag(rb, o.to_dist(xv, P))[rank])
        yv = comm.bcast(np.random.default_rng(2).standard_normal(sum(ny - r for r in range(P))).astype(dtype), 0)
        check("bd2H", host((BD2.H @ pm.DistributedArray.to_dist(yv)).local_array),
              o.blockdiag(rb, o.to_dist(yv, P), adjoint=True)[rank])
        VS2 = pm.MPIVStack([pm.MatrixMult(rb[rank][0])])
        check("vs2H", host((VS2.H @ pm.DistributedArray.to_dist(yv)).local_array), o.vstack_rmatvec(rb, o.to_dist(yv, P)), 1e-11, 1e-11)

# ---- MPIMatrixMult (square grids only, like the reference) -------------------------------------------
Pp = math.isqrt(P)
if Pp * Pp == P:
    for (N, K, M, dtype) in [(64, 64, 64, np.float64), (37, 37, 37, np.float64), (50, 30, 40, np.float64),
                             (22, 20, 16, np.complex128), (13, 14, 15, np.float32), (64, 48, Pp, np.float64)]:
        A = np.arange(N * K, dtype=dtype).reshape(N, K)
        X = np.arange(K * M, dtype=dtype).reshape(K, M)
        if dtype is np.complex128:
            A, X = A + 0.5j * A, X + 0.7j * X
        rtol = np.finfo(dtype).resolution * 10
        Yref = A.astype(np.complex128 if np.iscomplexobj(A) else np.float64) @ X
        # SUMMA: 2-D tiles (test_matrixmult.py:108-127)
        rs, cs = pm.local_block_split((N, K), rank, comm)
        assert (rs, cs) == o.local_block_split((N, K), rank, P)
        Aop = pm.MPIMatrixMult(A[rs, cs].copy(), M, kind="summa", dtype=dtype)
        xs = pm.local_block_split((K, M), rank, comm)
        sizes = [int(np.prod(X[o.local_block_split((K, M), r, P)].shape)) for r in range(P)]
        xd = pm.DistributedArray(global_shape=K * M, local_shapes=sizes, dtype=dtype)
        xd[:] = X[xs].ravel()
        y = Aop @ xd
        At = o.summa_tiles(A, P)
        yo = o.summa_matvec(At, [t.flatten() for t in o.summa_tiles(X, P)], N, K, M, dtype=dtype)
        check("summa", host(y.local_array), yo[rank], rtol, 0)
        check("summa gather", host(pm.block_gather(y, (N, M), comm)), Yref, rtol, 0)
        xa = Aop.H @ y
        xo = o.summa_matvec(At, yo, N, K, M, dtype=dtype, adjoint=True)
        check("summaH", host(xa.local_array), xo[rank], rtol * 10, 0)
        # block variant (test_matrixmult.py:216-237)
        blk, bc = int(math.ceil(N / Pp)), int(math.ceil(M / Pp))
        ci, ri = rank % Pp, rank // Pp
        Arow = A[ci * blk:min(N, (ci + 1) * blk)].copy()
        Bop = pm.MPIMatrixMult(Arow, M, kind="block", dtype=dtype)
        Xc = X[:, ri * bc:min(M, (ri + 1) * bc)]
        ncs = [max(0, min(M, (r // Pp + 1) * bc) - (r // Pp) * bc) for r in range(P)]
        xd = pm.DistributedArray(global_shape=K * sum(ncs), local_shapes=[K * c for c in ncs], dtype=dtype)
        xd[:] = Xc.ravel()
        yb = Bop @ xd
        check("block", host(yb.local_array).reshape(N, -1), Yref[:, ri * bc:min(M, (ri + 1) * bc)], rtol, 0)
        xb = Bop.H @ yb
        check("blockH", host(xb.local_array).reshape(K, -1), (A.conj().T @ Yref)[:, ri * bc:min(M, (ri + 1) * bc)], rtol * 10, 0)

# ---- rectangular-grid SUMMA (extension; BASELINE config 4 uses 2 x 4): vs dense products ------------------
for (Pr, Pc) in [(g, P // g) for g in range(1, P + 1) if P % g == 0]:
    for (N, K, M, dtype) in [(64, 48, 40, np.float64), (37, 29, 23, np.float64), (24, 36, 16, np.complex128)]:
        A = comm.bcast(np.random.default_rng(11).standard_normal((N, K)), 0).astype(dtype)
        X = comm.bcast(np.random.default_rng(12).standard_normal((K, M)), 0).astype(dtype)
        if dtype is np.complex128:
            A, X = A + 0.5j * A[::-1], X - 0.25j * X[::-1]
        L = Pr * Pc // math.gcd(Pr, Pc)
        bn, bm = math.ceil(N / Pr), math.ceil(M / Pc)
        Kp = math.ceil(K / L) * L
        bkA, bkX = Kp // Pc, Kp // Pr
        ri, ci = divmod(rank, Pc)
        Aop = pm.MPIMatrixMult(A[ri * bn:(ri + 1) * bn, ci * bkA:(ci + 1) * bkA].copy(), M, kind="summa",
                               dtype=dtype, grid=(Pr, Pc))
        xt = [X[(r // Pc) * bkX:(r // Pc + 1) * bkX, (r % Pc) * bm:(r % Pc + 1) * bm] for r in range(P)]
        xd = pm.DistributedArray(global_shape=K * M, local_shapes=[t.size for t in xt], dtype=dtype)
        xd[:] = xt[rank].ravel()
        y = Aop @ xd
        Yref = A @ X
        check(f"rect summa {Pr}x{Pc}", host(y.local_array), Yref[ri * bn:(ri + 1) * bn, ci * bm:(ci + 1) * bm].ravel(), 1e-11, 1e-11)
        xa = Aop.H @ y
        Xref = A.conj().T @ Yref
        check(f"rect summaH {Pr}x{Pc}", host(xa.local_array), Xref[ri * bkX:(ri + 1) * bkX, ci * bm:(ci + 1) * bm].ravel(), 1e-10, 1e-10)
        Rop = pm.MPIMatrixMult(A[ri * bn:(ri + 1) * bn, ci * bkA:(ci + 1) * bkA].copy(), M, kind="summa",
                               dtype=dtype, grid=(Pr, Pc), replicate=True)
        yr = Rop @ xd
        check(f"replicated {Pr}x{Pc}", host(yr.local_array), host(y.local_array), 1e-11, 1e-11)
        check(f"replicatedH {Pr}x{Pc}", host((Rop.H @ yr).local_array), host(xa.local_array), 1e-10, 1e-10)

# ---- MPIFredholm1 (test_fredholm.py) -------------------------------------------------------------------
for nz in (5, 1):
    for dtype in (np.float64, np.complex64):
        cx = np.issubdtype(dtype, np.complexfloating)
        nsl, nx, ny = 21, 4, 6
        G = np.arange(nsl * nx * ny, dtype=np.float64).reshape(nsl, nx, ny)
        G = (G - 1j * G) if cx else G
        ext = [o.local_split((nsl,), P, r)[0] for r in range(P)]
        if 1 in ext:
            continue
        off = np.cumsum([0] + ext)
        G_loc = [G[off[r]:off[r + 1]] for r in range(P)]
        Fr = pm.MPIFredholm1(G_loc[rank].astype(dtype), nz=nz, dtype=dtype)
        xv = (np.ones((nsl, ny, nz)) + (1j if cx else 0)).astype(dtype)
        xd = pm.DistributedArray.to_dist(xv.ravel(), partition=pm.Partition.BROADCAST)
        y = Fr @ xd
        refy = o.fredholm1(G_loc, xv.ravel().astype(G.dtype), nz)
        check("fredholm", host(y.local_array), refy, 1e-5, 0)
        check("fredholmH", host((Fr.H @ y).local_array), o.fredholm1(G_loc, refy, nz, adjoint=True), 1e-4, 0)
        Ff = pm.MPIFredholm1(G_loc[rank].astype(dtype), nz=nz, dtype=dtype, fused=True)   # product + gather in one kernel
        for _ in range(3):   # repeated applies exercise the double-buffered peer arenas
            yf = Ff @ xd
            check("fredholm fused", host(yf.local_array), refy, 1e-5, 0)
            check("fredholmH fused", host((Ff.H @ yf).local_array), o.fredholm1(G_loc, refy, nz, adjoint=True), 1e-4, 0)

# ---- CGLS on BlockDiag (test_solver.py:150-196) vs oracle at the same P ---------------------------------
for ny, nx in [(11, 11), (31, 11)]:
    blocks = []
    for r in range(P):
        A = np.ones((ny, nx)) * (r + 1)
        blocks.append([A.T @ A + 1e-5 * np.eye(nx)])
    Op = pm.MPIBlockDiag([pm.MatrixMult(blocks[rank][0])])
    xt = comm.bcast(np.random.default_rng(42).normal(1, 10, P * nx), 0)
    y = Op @ pm.DistributedArray.to_dist(xt)
    xinv, istop, iit, r1, r2, cost = pm.cgls(Op, y, x0=pm.DistributedArray.to_dist(np.zeros(P * nx)), niter=nx, tol=1e-5)
    mv = lambda v: o.SimArray(o.blockdiag(blocks, v.locs))                  # noqa: E731
    rmv = lambda v: o.SimArray(o.blockdiag(blocks, v.locs, adjoint=True))   # noqa: E731
    xo, istop_o, iit_o, r1o, r2o, cost_o = o.cgls(mv, rmv, mv(o.SimArray(o.to_dist(xt, P))),
                                                  o.SimArray(o.to_dist(np.zeros(P * nx), P)), niter=nx, tol=1e-5)
    # Conditioning (tests/test_oracle.py::test_cgls_blockdiag_cost_is_rounding_noise_below_1e_6): after P iterations
    # the residual is ~1e-8 of its start = rounding noise; a 1-ulp perturbation of the ORACLE moves those cost entries
    # by > 10 % and the stopping iteration by one at P = 8.  Parity bound = 1e-6 of the problem scale.
    assert abs(iit - iit_o) <= 1, (iit, iit_o)
    kk = min(len(cost), len(cost_o))
    check("cgls x", host(xinv.local_array), xo.locs[rank], 1e-6, 1e-6 * np.abs(xt).max())
    check("cgls cost", np.asarray(cost[:kk]), np.asarray(cost_o[:kk]), 1e-6, 1e-6 * cost_o[0])

# ---- "next" rows: MPIGradient / stacked arrays (vs dense per-axis derivatives) ------------------------------------
for dims, samp in [((16 * P + 3, 11), (1.0, 0.5)), ((8 * P + 1, 6, 7), (0.4, 1.0, 2.0))]:
    for kind, edge in (("centered", True), ("forward", False)):
        n = int(np.prod(dims))
        xg = comm.bcast(rng.normal(0, 10, n), 0)
        Gop = pm.MPIGradient(dims, sampling=samp, kind=kind, edge=edge)
        yst = Gop.matvec(pm.DistributedArray.to_dist(xg))
        refs = [o.derivative_along_axis(xg.reshape(dims), ax, o.first_derivative_dense(dims[ax], samp[ax], kind, edge, 3))
                for ax in range(len(dims))]
        for ax in range(len(dims)):
            check(f"gradient {dims} ax{ax}", host(yst[ax].asarray()), refs[ax].ravel(), 1e-12, 1e-10)
        refa = sum(o.derivative_along_axis(refs[ax], ax, o.first_derivative_dense(dims[ax], samp[ax], kind, edge, 3).T)
                   for ax in range(len(dims)))
        check(f"gradientH {dims}", host(Gop.rmatvec(yst).asarray()), refa.ravel(), 1e-11, 1e-9)
        flat = np.concatenate([r.ravel() for r in refs])
        check("stacked dot", yst.dot(yst)[0], np.dot(flat, flat), 1e-12, 0)
        check("stacked norm", yst.norm()[0], np.linalg.norm(flat), 1e-12, 0)

# ---- "next" row: ISTA / FISTA on BlockDiag (fused one-pass update + one all-reduce per iteration) vs the oracle ---
import scipy.linalg  # noqa: E402
for solver, fn in (("ista", pm.ista), ("fista", pm.fista)):
    for kind, eps in (("soft", 0.5), ("hard", 0.05)):
        rs = np.random.default_rng(21)
        ny, nx = 13, 11
        blocks = [rs.standard_normal((ny, nx)) for _ in range(P)]
        xtrue = np.zeros(P * nx)
        xtrue[rs.permutation(P * nx)[:max(2, P * nx // 5)]] = rs.standard_normal(max(2, P * nx // 5)) * 3
        alpha = 1.0 / max(np.linalg.norm(b, 2) ** 2 for b in blocks)
        Op = pm.MPIBlockDiag([pm.MatrixMult(blocks[rank])])
        ysp = Op @ pm.DistributedArray.to_dist(xtrue)
        xs, its, cs = fn(Op, ysp, pm.DistributedArray.to_dist(np.zeros(P * nx)), niter=30, eps=eps, alpha=alpha,
                         tol=1e-10, threshkind=kind)
        Ad = scipy.linalg.block_diag(*blocks)
        xo, ito, co = o.ista(Ad, Ad @ xtrue, np.zeros(P * nx), 30, eps, alpha, 1e-10, kind, fista=(solver == "fista"))
        assert its == ito
        check(f"{solver} {kind} x", host(xs.asarray()), xo, 1e-9, 1e-9)
        check(f"{solver} {kind} cost", cs, co, 1e-9, 0)

# ---- round 2: the driver-visible parity set of bench.py (peer-memory halo, stationary-A / replicated / SUMMA bf16 on
#      every grid of P, tensor-core Fredholm incl. fused peer all-gather, CGLS graph replay) at this world size ------
sys.path.insert(0, os.path.join(ROOT, "tests"))
import parity_checks  # noqa: E402
res = parity_checks.run_all(pm, comm, full_size=(os.environ.get("B2_PARITY_FULL", "0") == "1"))
assert res["failed"] == 0, res["failures"]

# frequency-domain MDC (scattered spectrum) at P ranks: F1^H I1^H of its gathered output == time-domain MDC
import warnings  # noqa: E402
nt, ns, nr, nv = 8 * P + 8, 5, 6, 3        # one-sided: nfft = 4 P + 5 >= the 4 P slices of the band
nfmax = 4 * P
gt = comm.bcast(np.random.default_rng(31).standard_normal((nt, ns, nr)), 0)
Gf = np.fft.rfft(gt, n=nt, axis=0)[:nfmax].astype(np.complex128)
off = np.arange(P + 1) * 4
mt = comm.bcast(np.random.default_rng(32).standard_normal(nt * nr * nv), 0)
md = pm.DistributedArray.to_dist(mt, partition=pm.Partition.BROADCAST)
Mt = pm.MPIMDC(Gf[off[rank]:off[rank + 1]], nt=nt, nv=nv, nfreq=nfmax, dt=0.004, dr=2.0, twosided=False)
Mf = pm.MPIMDC(Gf[off[rank]:off[rank + 1]], nt=nt, nv=nv, nfreq=nfmax, dt=0.004, dr=2.0, twosided=False, data_domain="frequency")
G_loc = [Gf[off[r]:off[r + 1]] for r in range(P)]
dt_ = Mt @ md
check("mdc time", host(dt_.asarray()).real, o.mdc(G_loc, mt, nt, nv, False, False, dt=0.004, dr=2.0), 1e-10, 1e-10)
df = Mf @ md
assert df.partition is pm.Partition.SCATTER
spec = host(Mf.data_to_frequency(dt_).asarray())
got = host(df.asarray())
check("mdc frequency (non-DC bins)", got[ns * nv:], spec[ns * nv:], 1e-9, 1e-9 * np.abs(spec).max())
with warnings.catch_warnings():
    warnings.simplefilter("ignore")
    x0 = pm.DistributedArray.to_dist(np.zeros(nt * nr * nv), partition=pm.Partition.BROADCAST)
    xt_, *_ = pm.cgls(Mt, dt_, x0=x0, niter=6, tol=0.0)
    xf_, *_ = pm.cgls(Mf, Mf.data_to_frequency(dt_), x0=x0, niter=6, tol=0.0)
check("mdd iterates time vs frequency domain", host(xf_.asarray()).real, host(xt_.asarray()).real, 1e-6,
      1e-6 * np.abs(host(xt_.asarray())).max())

comm.Barrier()
torch.cuda.synchronize()
print(f"MULTI_WORKER_OK rank={rank} size={P}")
