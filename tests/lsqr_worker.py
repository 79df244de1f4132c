"""LSQR at world size P under torchrun (one process per GPU).  Started by tests/test_lsqr.py.

  - MPIBlockDiag (SCATTER model), rank r holding diagonal block r of a fixture case (P = 2 = NBLK): istop and the
    iteration count exactly, x, var, the scalars and the cost within the single-GPU tolerances of test_lsqr.py;
  - MPIVStack (BROADCAST model) of both blocks: against the same solve on a one-rank communicator in this process.
    Every rank updates the whole model but adds only its share to |dk|^2: a doubled ddnorm would move acond by a
    factor sqrt(2).  The scalars are allowed 0.1 (of themselves; r1norm, r2norm of cost[0], arnorm of anorm * cost[0]),
    x 1e-4 of its largest entry: the two solves differ in the order of the all-reduced sums only, and the damped
    fixture's spreads under a 4-ulp jitter per iteration are 1.2e-2 for acond and 7.7e-6 for x;
  - both: the graph-replayed run and a step() loop give identical bits at P = 2.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import pylops_mpi_b200 as pm  # noqa: E402
from pylops_mpi_b200.optimization.cls_basic import LSQR  # noqa: E402

comm = pm.get_comm_world()
rank, P = comm.Get_rank(), comm.Get_size()
import test_lsqr as T  # noqa: E402

mgl = T.mgl
assert P == mgl.NBLK, P
GOLD = T.GOLD


def host(t):
    return t.cpu().numpy()


def block(name, r):
    A = GOLD[f"{name}/A"]
    m, n = A.shape[0] // mgl.NBLK, A.shape[1] // mgl.NBLK
    return np.ascontiguousarray(A[r * m:(r + 1) * m, r * n:(r + 1) * n])


def step_loop(Op, y, x0, kw):
    s = LSQR(Op)
    x = s.setup(y=y, x0=x0, **kw)
    while s.iiter < kw["niter"] and s.istop == 0:
        x = s.step(x)
    s.finalize()
    return (x, s.istop, s.iiter, s.r1norm, s.r2norm, s.anorm, s.acond, s.arnorm, s.xnorm, s.var, s.cost)


def flat(out):
    return [host(o.asarray()) if hasattr(o, "asarray") else np.asarray(o) for o in out]


def same_bits(a, b, what):
    for i, (g, r) in enumerate(zip(flat(a), flat(b))):
        np.testing.assert_array_equal(g, r, err_msg=f"[rank {rank}] {what}: output {i}")


for name in ("inconsistent", "illcond", "damped", "complex"):
    kw, has_x0 = T.params(name)
    Op = pm.MPIBlockDiag([pm.MatrixMult(block(name, rank))])
    y = pm.DistributedArray.to_dist(GOLD[f"{name}/b"])
    x0 = pm.DistributedArray.to_dist(GOLD[f"{name}/x0"]) if has_x0 else None
    s = LSQR(Op)
    out = s.solve(y, x0, **kw)
    assert s.graph_error is None and s.graph_replays > 0, s.graph_error
    x, istop, itn, r1, r2, anorm, acond, arnorm, xnorm, var, cost = out
    assert istop == int(GOLD[f"{name}/istop"]) and itn == int(GOLD[f"{name}/itn"]), (rank, name, istop, itn)
    xg, vg = GOLD[f"{name}/x"], GOLD[f"{name}/var"]
    np.testing.assert_allclose(host(x.asarray()), xg, rtol=0, atol=T.tol(name, 0) * np.abs(xg).max())
    np.testing.assert_allclose(host(var.asarray()), vg, rtol=0, atol=T.tol(name, 1) * np.abs(vg).max())
    for i, (k, got) in enumerate(zip(T.SCALARS, (r1, r2, anorm, acond, arnorm, xnorm))):
        assert abs(got - float(GOLD[f"{name}/{k}"])) <= T.tol(name, 2 + i) * T.scalar_scale(name, k), (rank, name, k)
    cg = GOLD[f"{name}/cost"]
    np.testing.assert_allclose(cost, cg, rtol=0, atol=T.tol(name, 8) * cg[0])
    same_bits(step_loop(Op, y, x0, kw), out, f"blockdiag {name} step vs graph")

one = pm.Comm(rank=0, size=1)
for name in ("inconsistent", "damped"):
    kw, _ = T.params(name)
    kw["niter"] = min(kw["niter"], 40)
    blocks = [block(name, r) for r in range(P)]
    b = GOLD[f"{name}/b"]
    Op = pm.MPIVStack([pm.MatrixMult(blocks[rank])])
    y = pm.DistributedArray.to_dist(b)
    s = LSQR(Op)
    out = s.solve(y, None, **kw)
    assert s.graph_error is None and s.graph_replays > 0, s.graph_error
    same_bits(step_loop(Op, y, None, kw), out, f"vstack {name} step vs graph")
    Op1 = pm.MPIVStack([pm.MatrixMult(np.vstack(blocks))], base_comm=one)
    ref = pm.lsqr(Op1, pm.DistributedArray.to_dist(b, base_comm=one), niter=kw["niter"], damp=kw["damp"],
                  atol=kw["atol"], btol=kw["btol"], conlim=kw["conlim"])
    assert out[1] == ref[1] and out[2] == ref[2], (rank, name, out[1:3], ref[1:3])
    np.testing.assert_allclose(host(out[0].asarray()), host(ref[0].asarray()), rtol=0,
                               atol=1e-4 * np.abs(host(ref[0].asarray())).max(), err_msg=f"[rank {rank}] {name} x")
    c0 = float(ref[10][0])
    for i, k in enumerate(T.SCALARS):
        scale = {"r1norm": c0, "r2norm": c0, "arnorm": ref[5] * c0}.get(k, abs(ref[3 + i]))
        assert abs(out[3 + i] - ref[3 + i]) <= 0.1 * scale, (rank, name, k, out[3 + i], ref[3 + i])

comm.Barrier()
torch.cuda.synchronize()
print(f"LSQR_WORKER_OK rank={rank} size={P}")
