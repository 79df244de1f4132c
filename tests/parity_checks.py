"""Driver-visible multi-rank parity set (TEST INFRASTRUCTURE: imports the CPU oracle as the checker).

``bench.py --gpus N`` runs :func:`run_all` on every rank BEFORE any timing and reports
``"parity": {"checked": k, "failed": f, ...}`` in its JSON line: the driver's GPU test box has one GPU, so
this is where the P = 2 / 4 / 8 paths (NCCL collectives, peer-memory halo / all-reduce / all-gather kernels,
rectangular SUMMA grid, BlockDiag CGLS) are compared with the oracle simulating the reference at the SAME
world size.  Reference tests mirrored: tests/test_derivative.py:198-229, test_distributedarray.py:270-361,
test_matrixmult.py:82-166, test_fredholm.py:154-167, test_solver.py:150-196; the BASELINE-size checks follow
SURVEY.md section 8(d) (C4: sampled rows of the 32768^2 bf16 product, C5: 64 x 256 x 256 x 64 complex64).

Every check returns (name, ok, detail); nothing here is timed.
"""
from __future__ import annotations

import math
import os
import sys
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "oracle")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402


def _host(t):
    return t.cpu().numpy()


def _close(got, ref, rtol, atol):
    got, ref = np.asarray(got), np.asarray(ref)
    if got.shape != ref.shape:
        return False, f"shape {got.shape} != {ref.shape}"
    err = np.abs(got - ref)
    tol = atol + rtol * np.abs(ref)
    bad = err > tol
    if bad.any():
        i = int(np.argmax(err - tol))
        return False, f"max violation at {i}: got {got.ravel()[i]!r} ref {ref.ravel()[i]!r}"
    return True, f"max abs err {float(err.max()) if err.size else 0.0:.3e}"


def run_all(pm, comm, full_size: bool = True):
    """returns {"checked": k, "failed": f, "failures": [...], "names": [...]} (identical on every rank)"""
    import torch
    import pylops_mpi_oracle as o
    rank, P = comm.Get_rank(), comm.Get_size()
    results = []

    def check(name, fn):
        try:
            ok, detail = fn()
        except Exception as exc:       # a crash is a failure of that check, not of the bench
            ok, detail = False, "".join(traceback.format_exception_only(type(exc), exc)).strip()[:300]
        results.append((name, bool(ok), detail))

    # ---- config 1: MPIFirstDerivative (11 x 21) float64 at P = world size (README.md:73-94) ------------------
    def fd_config1():
        x = np.zeros((11, 21))
        x[5, 10] = 1.0
        Fop = pm.MPIFirstDerivative((11, 21), dtype=np.float64)
        y = Fop @ pm.DistributedArray.to_dist(x.ravel())
        e = np.zeros((11, 21))
        e[4, 10], e[6, 10] = 0.5, -0.5
        got = _host(y.asarray())
        if not np.array_equal(got, e.ravel()):
            return False, "KAT mismatch"
        try:       # per-rank blocks vs the reference's own split (the reference cannot split 11 rows over 8 ranks)
            refl = o.first_derivative(o.to_dist(x.ravel(), P), (11, 21))
            if not np.array_equal(_host(y.local_array), refl[rank]):
                return False, "per-rank block differs from the oracle"
        except (ValueError, IndexError):
            pass
        u = pm.DistributedArray.to_dist(comm.bcast(np.random.default_rng(42).normal(0, 10, 231), 0))
        v = pm.DistributedArray.to_dist(comm.bcast(np.random.default_rng(43).normal(0, 10, 231), 0))
        return bool(pm.dottest(Fop, u, v)), "KAT + dottest"
    check("C1 MPIFirstDerivative (11,21) f64 KAT/per-rank/dottest", fd_config1)

    # ---- stencil grid at P ranks (fused peer-memory halo path when rows >= 2 per rank) vs dense D, D^T --------
    def fd_grid():
        rng = np.random.default_rng(7)
        worst = 0.0
        for dims, h in [((64 * P, 256), 1.0), ((16 * P + 3, 40), 0.4), ((8 * P + 1, 6, 16), 0.4)]:
            for kind, order in [("forward", 3), ("backward", 3), ("centered", 3), ("centered", 5)]:
                for edge in (False, True):
                    n = int(np.prod(dims))
                    xg = comm.bcast(rng.normal(0, 10, n), 0)
                    Fop = pm.MPIFirstDerivative(dims, sampling=h, kind=kind, edge=edge, order=order, dtype=np.float64)
                    D = o.first_derivative_dense(dims[0], h, kind, edge, order)
                    X = xg.reshape(dims[0], -1)
                    xd = pm.DistributedArray.to_dist(xg)
                    for _ in range(2):          # twice: both parities of the halo boxes
                        y, ya = Fop @ xd, Fop.H @ xd
                    for got, ref in ((y, D @ X), (ya, D.T @ X)):
                        ok, det = _close(_host(got.asarray()), ref.ravel(), 1e-12, 1e-12)
                        if not ok:
                            return False, f"{dims} {kind}{order} edge={edge}: {det}"
                        worst = max(worst, float(det.split()[-1]))
            Sop = pm.MPISecondDerivative(dims, sampling=h, kind="centered", edge=True, dtype=np.float64)
            D2 = o.second_derivative_dense(dims[0], h, "centered", True)
            xg = comm.bcast(rng.normal(0, 10, int(np.prod(dims))), 0)
            xd = pm.DistributedArray.to_dist(xg)
            for got, ref in ((Sop @ xd, D2 @ xg.reshape(dims[0], -1)), (Sop.H @ xd, D2.T @ xg.reshape(dims[0], -1))):
                ok, det = _close(_host(got.asarray()), ref.ravel(), 1e-12, 1e-10)
                if not ok:
                    return False, f"second derivative {dims}: {det}"
        return True, f"worst abs err {worst:.2e}"
    check("MPIFirst/SecondDerivative grid vs dense stencil matrices (halo over peer memory)", fd_grid)

    # ---- masked dot / norm (test_distributedarray.py:270-361) ---------------------------------------------
    def masked():
        if P < 2:
            return True, "skipped at P=1"
        mask = [r % 2 for r in range(P)]
        x = np.arange(24.0 * P) - 5.0
        X = pm.DistributedArray.to_dist(x, mask=mask)
        xl = o.to_dist(x, P)
        ok1, d1 = _close(X.dot(X)[0], o.dot(xl, xl, mask=mask)[rank], 1e-14, 0)
        ok2, d2 = _close(X.norm(1)[0], o.norm(xl, 1, mask=mask)[rank], 1e-14, 0)
        ok3, d3 = _close(X.norm(np.inf)[0], o.norm(xl, np.inf, mask=mask)[rank], 1e-14, 0)
        return ok1 and ok2 and ok3, f"{d1}; {d2}; {d3}"
    check("masked dot / norm on sub-communicators", masked)

    # ---- dot / norm on float32 SCATTER vectors vs float64 oracle (config 2 parity bound) ---------------------
    def reductions():
        n = 100003
        xs = [np.random.default_rng(42 + r).standard_normal(n).astype(np.float32) for r in range(P)]
        ys = [np.random.default_rng(142 + r).standard_normal(n).astype(np.float32) for r in range(P)]
        X = pm.DistributedArray(global_shape=n * P, dtype=np.float32)
        Y = pm.DistributedArray(global_shape=n * P, dtype=np.float32)
        X[:] = xs[rank]
        Y[:] = ys[rank]
        d_ref = sum(np.dot(a.astype(np.float64), b.astype(np.float64)) for a, b in zip(xs, ys))
        scale = math.sqrt(sum(np.dot(a.astype(np.float64), a.astype(np.float64)) for a in xs) *
                          sum(np.dot(b.astype(np.float64), b.astype(np.float64)) for b in ys))
        tol = max(1e-6, 4 * np.finfo(np.float32).eps * math.sqrt(n * P))
        ok1 = abs(float(X.dot(Y)[0]) - d_ref) <= tol * scale
        n2 = math.sqrt(sum(np.dot(a.astype(np.float64), a.astype(np.float64)) for a in xs))
        ok2, d2 = _close(X.norm()[0], n2, 1e-6, 0)
        ok3, d3 = _close(X.norm(1)[0], sum(np.abs(a.astype(np.float64)).sum() for a in xs), 1e-6, 0)
        ok4, d4 = _close(X.norm(np.inf)[0], max(np.abs(a).max() for a in xs), 0, 0)
        return ok1 and ok2 and ok3 and ok4, f"dot rel {abs(float(X.dot(Y)[0]) - d_ref) / scale:.2e}; {d2}; {d3}; {d4}"
    check("C2 dot / norm float32 vs float64 oracle", reductions)

    # ---- array all-reduce (peer-memory one-shot path and NCCL path): exact integer sums ----------------------
    def allreduce():
        from pylops_mpi_b200.Distributed import allreduce_
        for dt in (torch.float32, torch.float64):
            for nel in (1, 9, 1000, 16384, 70001, 300000):
                gen = torch.Generator(device="cuda").manual_seed(1234 + rank)
                v = torch.randint(-1000, 1000, (nel,), device="cuda", generator=gen).to(dt)
                ref = torch.zeros(nel, dtype=dt, device="cuda")
                for r in range(P):
                    g2 = torch.Generator(device="cuda").manual_seed(1234 + r)
                    ref += torch.randint(-1000, 1000, (nel,), device="cuda", generator=g2).to(dt)
                for _ in range(3):
                    w = v.clone()
                    allreduce_(comm, w)
                    if not torch.equal(w, ref):
                        return False, f"{dt} n={nel}"
        return True, "exact"
    check("array Allreduce (VStack adjoint path), exact sums", allreduce)

    # ---- BlockDiag / VStack KATs (test_blockdiag.py:24-71, test_stack.py:29-79) ------------------------------
    def stacks():
        ny, nx = 301, 101
        for dtype in (np.float64, np.complex128):
            blk = ((rank + 1) * np.ones((ny, nx))).astype(dtype)
            BD = pm.MPIBlockDiag([pm.MatrixMult(blk)])
            xd = pm.DistributedArray(global_shape=P * nx, dtype=dtype)
            xd[:] = 1.0
            ok, det = _close(_host((BD @ xd).local_array), (rank + 1) * nx * np.ones(ny), 1e-13, 0)
            if not ok:
                return False, "blockdiag " + det
            yd = pm.DistributedArray(global_shape=P * ny, dtype=dtype)
            yd[:] = 1.0
            VS = pm.MPIVStack([pm.MatrixMult(blk)])
            xr = VS.H @ yd
            ok, det = _close(_host(xr.local_array), sum(r + 1 for r in range(P)) * ny * np.ones(nx), 1e-13, 0)
            if not ok:
                return False, "vstack adjoint " + det
        return True, "ones blocks"
    check("MPIBlockDiag / MPIVStack KATs", stacks)

    # ---- SUMMA on the BASELINE grid shape (rectangular Pr x Pc), float64, vs dense ---------------------------
    def summa_rect():
        grids = {1: (1, 1), 2: (1, 2), 4: (2, 2), 8: (2, 4)}
        if P not in grids:
            return True, f"no grid for P={P}"
        Pr, Pc = grids[P]
        worst = 0.0
        for (N, K, M) in [(64, 48, 40), (37, 29, 23)]:
            A = comm.bcast(np.random.default_rng(11).standard_normal((N, K)), 0)
            X = comm.bcast(np.random.default_rng(12).standard_normal((K, M)), 0)
            L = Pr * Pc // math.gcd(Pr, Pc)
            bn, bm = math.ceil(N / Pr), math.ceil(M / Pc)
            Kp = math.ceil(K / L) * L
            bkA, bkX = Kp // Pc, Kp // Pr
            ri, ci = divmod(rank, Pc)
            xt = [X[(r // Pc) * bkX:(r // Pc + 1) * bkX, (r % Pc) * bm:(r % Pc + 1) * bm] for r in range(P)]
            Yref = A @ X
            Xref = A.T @ Yref
            for kw in ({}, {"replicate": True}):
                Aop = pm.MPIMatrixMult(A[ri * bn:(ri + 1) * bn, ci * bkA:(ci + 1) * bkA].copy(), M, kind="summa",
                                       dtype=np.float64, grid=(Pr, Pc), **kw)
                xd = pm.DistributedArray(global_shape=K * M, local_shapes=[t.size for t in xt], dtype=np.float64)
                xd[:] = xt[rank].ravel()
                y = Aop @ xd
                ok, det = _close(_host(y.local_array), Yref[ri * bn:(ri + 1) * bn, ci * bm:(ci + 1) * bm].ravel(), 1e-11, 1e-11)
                if not ok:
                    return False, f"{kw} forward {det}"
                xa = Aop.H @ y
                ok, det = _close(_host(xa.local_array), Xref[ri * bkX:(ri + 1) * bkX, ci * bm:(ci + 1) * bm].ravel(), 1e-10, 1e-10)
                if not ok:
                    return False, f"{kw} adjoint {det}"
                worst = max(worst, float(det.split()[-1]))
        return True, f"grid {Pr}x{Pc}, worst {worst:.2e}"
    check("MPIMatrixMult SUMMA on the BASELINE grid (float64) vs dense", summa_rect)

    # ---- bf16 -> fp32 tensor-core modes on every factorisation of P: SUMMA / replicated / stationary-A ------------
    def summa_bf16_modes():
        worst = 0.0
        for (Pr, Pc) in [(g, P // g) for g in range(1, P + 1) if P % g == 0]:
            L = Pr * Pc // math.gcd(Pr, Pc)
            # ragged N and K (zero-padding paths) whose padded tiles stay 8-aligned; M / Pc % 32 == 0
            N, K, M = 64 * Pr - (1 if Pr > 1 else 0), 128 * L - (1 if L > 1 else 0), 64 * Pc
            bn, bm = math.ceil(N / Pr), math.ceil(M / Pc)
            Kp = math.ceil(K / L) * L
            bkA, bkX = Kp // Pc, Kp // Pr
            A = comm.bcast(np.random.default_rng(21).standard_normal((N, K)).astype(np.float32) / 16, 0)
            X = comm.bcast(np.random.default_rng(22).standard_normal((K, M)).astype(np.float32), 0)
            Ab = torch.as_tensor(A).to(torch.bfloat16)
            A64 = Ab.double().numpy()
            Xb = torch.as_tensor(X).to(torch.bfloat16).double().numpy()
            ri, ci = divmod(rank, Pc)
            xt = [X[(r // Pc) * bkX:(r // Pc + 1) * bkX, (r % Pc) * bm:(r % Pc + 1) * bm] for r in range(P)]
            Yref = A64 @ Xb
            bound = (np.abs(A64) @ np.abs(Xb)) * K * 6e-8 + 1e-6
            for kw in ({}, {"replicate": True}, {"stationary": True}):
                try:
                    Aop = pm.MPIMatrixMult(Ab[ri * bn:(ri + 1) * bn, ci * bkA:(ci + 1) * bkA].contiguous(), M,
                                           kind="summa", dtype="bfloat16", grid=(Pr, Pc), **kw)
                except NotImplementedError as exc:
                    if "stationary" in kw:
                        continue        # tile extents of this factorisation are not 8 / 32-aligned
                    raise exc
                xd = pm.DistributedArray(global_shape=K * M, local_shapes=[t.size for t in xt], dtype=np.float32)
                xd[:] = xt[rank].ravel()
                for _ in range(2):
                    y = Aop @ xd
                got = _host(y.local_array).reshape(-1, min(bm, M - ci * bm))
                ref = Yref[ri * bn:(ri + 1) * bn, ci * bm:(ci + 1) * bm]
                if got.shape != ref.shape or not np.all(np.abs(got - ref) <= bound[ri * bn:(ri + 1) * bn, ci * bm:(ci + 1) * bm]):
                    return False, f"grid {Pr}x{Pc} {kw or 'summa'} forward"
                worst = max(worst, float(np.abs(got - ref).max()))
                # adjoint of the (bf16-rounded, as the operator does) forward result
                Yb = torch.as_tensor(Yref.astype(np.float32)).to(torch.bfloat16).double().numpy()
                yt = [Yref[(r // Pc) * bn:(r // Pc + 1) * bn, (r % Pc) * bm:(r % Pc + 1) * bm] for r in range(P)]
                yd = pm.DistributedArray(global_shape=N * M, local_shapes=[t.size for t in yt], dtype=np.float32)
                yd[:] = yt[rank].astype(np.float32).ravel()
                xa = Aop.H @ yd
                Xref = A64.T @ Yb
                bounda = (np.abs(A64.T) @ np.abs(Yb)) * N * 6e-8 + 1e-4
                gota = _host(xa.local_array).reshape(-1, min(bm, M - ci * bm))
                refa = Xref[ri * bkX:(ri + 1) * bkX, ci * bm:(ci + 1) * bm]
                if gota.shape != refa.shape or not np.all(np.abs(gota - refa) <= bounda[ri * bkX:(ri + 1) * bkX, ci * bm:(ci + 1) * bm]):
                    return False, f"grid {Pr}x{Pc} {kw or 'summa'} adjoint"
        return True, f"all grids of P={P}, worst abs err {worst:.2e}"
    check("MPIMatrixMult bf16->fp32: SUMMA / replicated / stationary-A on every grid vs float64", summa_bf16_modes)

    # ---- Fredholm1 KAT (test_fredholm.py:36-95), SIMT, tensor-core and fused peer paths -----------------------
    def fredholm_kat():
        F1 = pm.signalprocessing.Fredholm1
        nsl, nx, ny = 21, 4, 6
        ext = [o.local_split((nsl,), P, r)[0] for r in range(P)]
        if 1 in ext or 0 in ext:
            return True, f"reference rejects this split at P={P}"
        off = np.cumsum([0] + ext)
        for nz in (5, 1):
            for dtype in (np.float64, np.complex64):
                cx = np.issubdtype(dtype, np.complexfloating)
                G = np.arange(nsl * nx * ny, dtype=np.float64).reshape(nsl, nx, ny)
                G = (G - 1j * G) if cx else G
                G_loc = [G[off[r]:off[r + 1]] for r in range(P)]
                xv = (np.ones((nsl, ny, nz)) + (1j if cx else 0)).astype(dtype)
                refy = o.fredholm1(G_loc, xv.ravel().astype(G.dtype), nz)
                refx = o.fredholm1(G_loc, refy, nz, adjoint=True)
                xd = pm.DistributedArray.to_dist(xv.ravel(), partition=pm.Partition.BROADCAST)
                # the default threshold keeps these shapes on the SIMT kernel, threshold 0 puts complex64 on the plan
                for tc_min in (F1.TC_MIN_PRODUCTS, 0):
                    saved, F1.TC_MIN_PRODUCTS = F1.TC_MIN_PRODUCTS, tc_min
                    try:
                        for fused in (False, True) if P > 1 else (False,):
                            Fr = pm.MPIFredholm1(G_loc[rank].astype(dtype), nz=nz, dtype=dtype, fused=fused)
                            for _ in range(2):
                                y = Fr @ xd
                                ok, det = _close(_host(y.local_array), refy, 1e-5, 0)
                                if not ok:
                                    return False, f"nz={nz} {dtype.__name__} tc_min={tc_min} fused={fused}: {det}"
                                ok, det = _close(_host((Fr.H @ y).local_array), refx, 1e-4, 0)
                                if not ok:
                                    return False, f"adjoint nz={nz} {dtype.__name__} tc_min={tc_min} fused={fused}: {det}"
                    finally:
                        F1.TC_MIN_PRODUCTS = saved
        return True, "arange KAT"
    check("MPIFredholm1 arange KAT (SIMT / tensor cores / fused peer all-gather)", fredholm_kat)

    # ---- C5 at BASELINE size: 64 slices/GPU of 256 x 256 x 64 complex64 vs complex128 -----------------------
    def fredholm_full():
        nsl, ns, nr, nv = 64, 256, 256, 64
        g = torch.Generator(device="cuda").manual_seed(3 + rank)
        G = torch.randn(nsl, ns, nr, device="cuda", dtype=torch.complex64, generator=g)
        Fr = pm.MPIFredholm1(G, nz=nv, dtype=np.complex64)
        xm = pm.DistributedArray(global_shape=nsl * P * nr * nv, partition=pm.Partition.BROADCAST, dtype=np.complex64)
        gx = torch.Generator(device="cuda").manual_seed(4)
        xm.local_array.copy_(torch.randn(nsl * P * nr * nv, device="cuda", dtype=torch.complex64, generator=gx))
        y = Fr @ xm
        ya = Fr.H @ y
        torch.cuda.synchronize()
        # this rank's slices against a complex128 product of the same inputs (every rank checks its own part)
        xs = xm.local_array.view(nsl * P, nr, nv)[rank * nsl:(rank + 1) * nsl].to(torch.complex128)
        ref = torch.matmul(G.to(torch.complex128), xs)
        got = y.local_array.view(nsl * P, ns, nv)[rank * nsl:(rank + 1) * nsl].to(torch.complex128)
        e1 = ((got - ref).abs().max() / ref.abs().max()).item()
        refa = torch.matmul(G.to(torch.complex128).conj().transpose(1, 2),
                            y.local_array.view(nsl * P, ns, nv)[rank * nsl:(rank + 1) * nsl].to(torch.complex128))
        gota = ya.local_array.view(nsl * P, nr, nv)[rank * nsl:(rank + 1) * nsl].to(torch.complex128)
        e2 = ((gota - refa).abs().max() / refa.abs().max()).item()
        # the gathered output must be identical on every rank (BROADCAST): compare a checksum
        cs = float(y.local_array.abs().double().sum().item())
        allcs = comm.allgather(cs)
        same = all(c == allcs[0] for c in allcs)
        return e1 < 1e-5 and e2 < 1e-5 and same, f"fwd {e1:.2e} adj {e2:.2e} (bound 1e-5 of max), broadcast identical={same}"
    if full_size:
        check("C5 MPIFredholm1 64x256x256x64 complex64 vs complex128 (rtol 1e-5 of max)", fredholm_full)

    # ---- config 3 flavour: CGLS on BlockDiag vs oracle.cgls at the same P (test_solver.py:150-196) ------------
    def cgls_blockdiag():
        out = []
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
            # Conditioning (tests/test_oracle.py::test_cgls_blockdiag_cost_is_rounding_noise_below_1e-6): the operator has
            # P distinct large eigenvalues and a 1e-5 cluster, so after P iterations the residual sits at ~1e-8 of its
            # start and is pure rounding noise -- a 1-ulp perturbation of the oracle itself moves those cost entries by
            # > 100 % and the stopping iteration by one.  Entries above 1e-6 of cost[0] must agree to 1e-6 relative;
            # below, to 1e-6 * cost[0] absolute; the iteration count may differ by one.
            if abs(iit - iit_o) > 1:
                return False, f"iterations {iit} vs {iit_o}"
            k = min(len(cost), len(cost_o))
            c, co = np.asarray(cost[:k]), np.asarray(cost_o[:k])
            ok, det = _close(c, co, 1e-6, 1e-6 * co[0])
            if not ok:
                return False, f"cost ({ny},{nx}): {det}"
            ok, det = _close(_host(xinv.local_array), xo.locs[rank], 1e-6, 1e-6 * np.abs(xt).max())
            if not ok:
                return False, f"x ({ny},{nx}): {det}"
            out.append(det)
        return True, "; ".join(out)
    check("CGLS on MPIBlockDiag vs oracle.cgls (1e-6 of the problem scale)", cgls_blockdiag)

    # ---- config 3 at BASELINE size: P x (4096 x 4096) float32 blocks, 50 iterations ---------------------------
    def cgls_full():
        nb = 4096
        A = torch.randn(nb, nb, device="cuda", generator=torch.Generator(device="cuda").manual_seed(100 + rank)) / 128
        A += 2 * torch.eye(nb, device="cuda")
        Op = pm.MPIBlockDiag([pm.MatrixMult(A)])
        xt = pm.DistributedArray(global_shape=nb * P, dtype=np.float32)
        xt.local_array.copy_(torch.randn(nb, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7 + rank)))
        yd = Op.matvec(xt)
        xinv, istop, iit, r1, r2, cost = pm.cgls(Op, yd, x0=xt.zeros_like(), niter=50, tol=0.0)
        err = float((xinv - xt).norm()[0] / xt.norm()[0])
        mono = bool(np.all(np.diff(cost[:20]) < 0))
        return err < 1e-5 and iit == 50 and mono, f"rel err vs x_true {err:.2e} after {iit} iterations"
    if full_size:
        check("C3 CGLS 50 it on P x (4096x4096) f32 BlockDiag converges to x_true (< 1e-5)", cgls_full)

    failed = [(n, d) for n, ok, d in results if not ok]
    # agree across ranks (a check may fail on one rank only)
    nfail = comm.allreduce(len(failed), "max") if P > 1 else len(failed)
    allfail = comm.allgather([f"[rank {rank}] {n}: {d}" for n, d in failed]) if P > 1 else [[f"{n}: {d}" for n, d in failed]]
    return {"checked": len(results), "failed": int(nfail), "world_size": P,
            "failures": [f for fl in allfail for f in fl][:8],
            "details": {n: d for n, ok, d in results}}


def sampled_rows_check(pm, comm, Sop, At_seed_fn, xs, y, Ng, Kg, Mg, Pr, Pc, nrows=256):
    """C4 at BASELINE size (SURVEY 8d): `nrows` sampled rows of this rank's output tile of the 32768^2 bf16
    product against a float64 product of the SAME bf16-rounded inputs.  Tiles of A and X are regenerated from
    their seeds (every rank can rebuild any tile), so no extra communication is needed.
    Bound: fp32 accumulation of K exact bf16 x bf16 products: |err| <= 1e-6 * sqrt(K) * ||a_row|| * ||x_col||."""
    import torch
    rank = comm.Get_rank()
    ri, ci = divmod(rank, Pc)
    bn, bkA, bkX, bm = Ng // Pr, Kg // Pc, Kg // Pr, Mg // Pc
    g = torch.Generator(device="cuda").manual_seed(99)
    rows = torch.randperm(bn, device="cuda", generator=g)[:nrows]
    # A[rows of grid row ri, all K] from the Pc tiles of that grid row
    Arow = torch.cat([At_seed_fn(ri * Pc + c)[rows] for c in range(Pc)], dim=1).to(torch.float64)        # nrows x Kg
    # X[:, columns of grid column ci] from the Pr tiles of that grid column (bf16-rounded like the operator does)
    Xcol = torch.cat([xs(r * Pc + ci) for r in range(Pr)], dim=0).to(torch.bfloat16).to(torch.float64)   # Kg x bm
    ref = Arow @ Xcol
    got = y.local_array.view(bn, bm)[rows].to(torch.float64)
    bound = 1e-6 * math.sqrt(Kg) * Arow.norm(dim=1, keepdim=True) * Xcol.norm(dim=0, keepdim=True)
    viol = ((got - ref).abs() / bound).max().item()
    rel = ((got - ref).norm() / ref.norm()).item()
    return viol <= 1.0, f"{nrows} rows: max |err|/bound {viol:.3f}, normwise rel {rel:.2e}"
