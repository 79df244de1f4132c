"""PoststackLinearModelling at world size P under torchrun (one process per GPU): each rank's MPIBlockDiag block
against its slice of the gathered reference fixtures of tests/golden/poststack_golden.npz, and the three solves of
tutorials/poststack.py against their fixtures.  Started by tests/test_poststack.py."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import make_golden_poststack as mgp  # noqa: E402
import pylops_mpi_b200 as pm  # noqa: E402

comm = pm.get_comm_world()
rank, P = comm.Get_rank(), comm.Get_size()
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "poststack_golden.npz"), allow_pickle=False)


def block(ny):
    """this rank's rows of y: (local_shapes, flat slice, local rows)"""
    rows = mgp.rows_of(P, ny)
    plane = mgp.NX * mgp.NT0
    lo, hi = sum(rows[:rank]) * plane, sum(rows[:rank + 1]) * plane
    return [(r * plane,) for r in rows], slice(lo, hi), rows[rank]


def local_op(layout, ny_r, wav, kind):
    PPop = pm.local.PoststackLinearModelling(wav, nt0=mgp.NT0, spatdims=(ny_r, mgp.NX), kind=kind)
    if layout == "native":
        return PPop
    Top = pm.local.Transpose((ny_r, mgp.NX, mgp.NT0), (2, 0, 1))
    return Top.H @ PPop @ Top


def host(t):
    return t.cpu().numpy()


def check(name, got, ref, rtol, atol):
    np.testing.assert_allclose(got, ref, rtol=rtol, atol=atol, err_msg=f"[rank {rank}] {name}")


ls, sl, ny_r = block(mgp.NY)
for (layout, Pc, kind, nh, dt) in mgp.cases():
    if Pc != P:
        continue
    wav, x, v = mgp.case_inputs(nh, dt)
    Op = pm.MPIBlockDiag([local_op(layout, ny_r, wav, kind)], dtype=dt)
    gy, gya = mgp.expected(GOLD, layout, P, kind, nh, dt)       # exact: the inputs are exactly representable
    name = f"{mgp.key(layout, P, kind, nh)}/{dt}"
    np.testing.assert_array_equal(host((Op @ pm.DistributedArray.to_dist(x, local_shapes=ls)).local_array), gy[sl],
                                  err_msg=f"[rank {rank}] {name}/y")
    np.testing.assert_array_equal(host((Op.H @ pm.DistributedArray.to_dist(v, local_shapes=ls)).local_array),
                                  gya[sl], err_msg=f"[rank {rank}] {name}/ya")

ls, sl, ny_i = block(mgp.FLOW_NY)
wav, m3d, mback3d = mgp.flow_inputs()
nx, nz = mgp.NX, mgp.NT0
PPop = pm.local.PoststackLinearModelling(wav, nt0=nz, spatdims=(ny_i, nx))
Top = pm.local.Transpose((ny_i, nx, nz), (2, 0, 1))
BDiag = pm.MPIBlockDiag([Top.H @ PPop @ Top])
m = pm.DistributedArray.to_dist(m3d.ravel(), local_shapes=ls)
x0 = pm.DistributedArray.to_dist(mback3d.ravel(), local_shapes=ls)
d = BDiag @ m
check("flow/d", host(d.local_array), GOLD["flow/d"][sl], 1e-12, 1e-12)


def check_flow(name, x, iiter, cost):
    g = f"flow/P{P}/{name}"
    assert iiter == int(GOLD[f"{g}/iiter"])
    check(f"{g}/cost", np.asarray(cost), GOLD[f"{g}/cost"], 1e-10, 0)
    check(f"{g}/x", host(x.local_array), GOLD[f"{g}/x"][sl], 1e-9, 1e-11)


x, _, iiter, _, _, cost = pm.cgls(BDiag, d, x0=x0, niter=mgp.FLOW_NITER, tol=0.0)
check_flow("iter", x, iiter, cost)
LapOp = pm.MPILaplacian(dims=(mgp.FLOW_NY, nx, nz), axes=(0, 1, 2), weights=(1, 1, 1), sampling=(1, 1, 1),
                        dtype=BDiag.dtype)
x, iiter, cost = pm.cg(BDiag.H @ BDiag + mgp.FLOW_EPSR * LapOp.H @ LapOp, BDiag.H @ d, x0=x0,
                       niter=mgp.FLOW_NITER, tol=0.0)
check_flow("ne", x, iiter, cost)
zero = pm.DistributedArray.to_dist(np.zeros(m3d.size), local_shapes=ls)
x, _, iiter, _, _, cost = pm.cgls(pm.MPIStackedVStack([BDiag, np.sqrt(mgp.FLOW_EPSR) * LapOp]),
                                  pm.StackedDistributedArray([d, zero]), x0=x0, niter=mgp.FLOW_NITER, tol=0.0)
check_flow("reg", x, iiter, cost)

comm.Barrier()
torch.cuda.synchronize()
print(f"POSTSTACK_WORKER_OK rank={rank} size={P}")
