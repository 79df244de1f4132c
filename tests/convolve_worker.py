"""Convolve1D at world size P under torchrun (one process per GPU): each rank's MPIBlockDiag([Convolve1D]) block
against its slice of the gathered reference fixtures of tests/golden/convolve_golden.npz, and the reflectivity ISTA
flow against its fixture.  Started by tests/test_convolve.py."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import make_golden_convolve as mgc  # noqa: E402
import pylops_mpi_b200 as pm  # noqa: E402

comm = pm.get_comm_world()
rank, P = comm.Get_rank(), comm.Get_size()
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "convolve_golden.npz"), allow_pickle=False)


def block(dims_global):
    """this rank's rows of a global array split along axis 0: (local_shapes, flat slice, local dims)"""
    rows = mgc.rows_of(P, dims_global)
    plane = int(np.prod(dims_global[1:]))
    lo, hi = sum(rows[:rank]) * plane, sum(rows[:rank + 1]) * plane
    return [(r * plane,) for r in rows], slice(lo, hi), (rows[rank],) + tuple(dims_global[1:])


def host(t):
    return t.cpu().numpy()


def check(name, got, ref, rtol, atol):
    np.testing.assert_allclose(got, ref, rtol=rtol, atol=atol, err_msg=f"[rank {rank}] {name}")


ls, sl, dims = block(mgc.DIMS)
for (Pc, axis, nh, off, dt) in mgc.cases():
    if Pc != P:
        continue
    h, x, v = mgc.case_inputs(nh, dt)
    Op = pm.MPIBlockDiag([pm.local.Convolve1D(dims, h, offset=off, axis=axis, dtype=dt)])
    gy, gya = mgc.expected(GOLD, P, axis, nh, off, dt)       # exact: the inputs are exactly representable
    name = f"{mgc.key(P, axis, nh, off)}/{dt}"
    np.testing.assert_array_equal(host((Op @ pm.DistributedArray.to_dist(x, local_shapes=ls)).local_array), gy[sl],
                                  err_msg=f"[rank {rank}] {name}/y")
    np.testing.assert_array_equal(host((Op.H @ pm.DistributedArray.to_dist(v, local_shapes=ls)).local_array),
                                  gya[sl], err_msg=f"[rank {rank}] {name}/ya")

ls, sl, dims = block(mgc.REFL_DIMS)
wav, m, alpha = mgc.refl_inputs()
DDiag = pm.MPIBlockDiag([pm.local.FirstDerivative(dims, axis=-1)])
CDiag = pm.MPIBlockDiag([pm.local.Convolve1D(dims, wav, offset=mgc.REFL_OFF, axis=-1)])
d = CDiag @ (DDiag @ pm.DistributedArray.to_dist(m, local_shapes=ls))
check("refl/d", host(d.local_array), GOLD["refl/d"][sl], 1e-12, 1e-12)
x0 = pm.DistributedArray.to_dist(np.zeros_like(m), local_shapes=ls)
x, iiter, cost = pm.ista(CDiag, d, x0, niter=mgc.REFL_NITER, eps=mgc.REFL_EPS, alpha=alpha, tol=1e-10)
assert iiter == int(GOLD[f"refl/P{P}/iiter"])
check("refl/cost", np.asarray(cost), GOLD[f"refl/P{P}/cost"], 1e-10, 0)
check("refl/x", host(x.local_array), GOLD[f"refl/P{P}/x"][sl], 1e-9, 1e-11)

comm.Barrier()
torch.cuda.synchronize()
print(f"CONVOLVE_WORKER_OK rank={rank} size={P}")
