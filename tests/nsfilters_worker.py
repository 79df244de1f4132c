"""NonStationaryFilters1D / 2D at world size P under torchrun (one process per GPU): each rank holds
MPIVStack([NonStationaryFilters(inp_k) for its inputs k]) with the bank broadcast, and the gathered forward and the
all-reduced adjoint must equal the reference fixtures of tests/golden/nsfilters_golden.npz bit for bit; then both
estimation flows' cgls at this P against their fixtures, within the recorded tolerances.  Started by
tests/test_nsfilters.py."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import make_golden_nsfilters as mgf  # noqa: E402
import pylops_mpi_b200 as pm  # noqa: E402

comm = pm.get_comm_world()
rank, P = comm.Get_rank(), comm.Get_size()
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "nsfilters_golden.npz"), allow_pickle=False)
rows = mgf.rows_of(P)
k0 = sum(rows[:rank])

for kind, nh, bank, dt in mgf.cases():
    inp, ih, _, x, v = mgf.case_inputs(kind, nh, bank, dt)
    plane = int(np.prod(inp.shape[1:]))
    mine = inp[k0:k0 + rows[rank]]
    ops = ([pm.local.NonStationaryFilters1D(i, nh, ih[0], dtype=dt) for i in mine] if kind == 1 else
           [pm.local.NonStationaryFilters2D(i, nh, *ih, dtype=dt) for i in mine])
    Op = pm.MPIVStack(ops, dtype=dt)
    ls = [(r * plane,) for r in rows]
    gy, gya = mgf.decode(GOLD, mgf.key(kind, nh, bank), dt)
    name = f"{mgf.key(kind, nh, bank)}/{dt}"
    y = (Op @ pm.DistributedArray.to_dist(x, partition=pm.Partition.BROADCAST)).local_array.cpu().numpy()
    np.testing.assert_array_equal(y, gy[k0 * plane:(k0 + rows[rank]) * plane], err_msg=f"[rank {rank}] {name}/y")
    ya = (Op.H @ pm.DistributedArray.to_dist(v, local_shapes=ls)).local_array.cpu().numpy()
    np.testing.assert_array_equal(ya, gya, err_msg=f"[rank {rank}] {name}/ya")

# the estimation flows: cgls over this rank's inputs, the bank all-reduced
for kind in (1, 2):
    f = f"flow{kind}"
    if kind == 1:
        inps, d, niter = GOLD["flow1/refl"], GOLD["flow1/d"], mgf.FLOW1_NITER
    else:
        inps, niter = GOLD["flow2/mmig"][:mgf.FLOW2_NTRAIN], mgf.FLOW2_NITER
        d = GOLD["flow2/m"][:mgf.FLOW2_NTRAIN].ravel()
    fr = mgf.rows_of(P, len(inps))
    f0 = sum(fr[:rank])
    plane = int(np.prod(inps.shape[1:]))
    ops = [pm.local.NonStationaryFilters1D(i, 15, mgf.FLOW1_IH) if kind == 1 else
           pm.local.NonStationaryFilters2D(i, mgf.FLOW2_NH, mgf.mg2.FLOW_IHX, mgf.mg2.FLOW_IHZ)
           for i in inps[f0:f0 + fr[rank]]]
    Op = pm.MPIVStack(ops)
    x0 = pm.DistributedArray.to_dist(np.zeros(Op.shape[1]), partition=pm.Partition.BROADCAST)
    dd = pm.DistributedArray.to_dist(d, local_shapes=[(r * plane,) for r in fr])
    x, _, iiter, _, _, cost = pm.cgls(Op, dd, x0=x0, niter=niter, tol=0.0)
    assert iiter == int(GOLD[f"{f}/P{P}/iiter"])
    floor = 10 * float(GOLD[f"{f}/cond"]) * 2.0 ** -53          # as tests/test_nsfilters.py's flow_tolerance()
    xtol, ctol = (max(100 * float(s), floor) for s in GOLD[f"{f}/spread"])
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"{f}/P{P}/cost"], rtol=ctol, err_msg=f"[rank {rank}] {f} cost")
    gx = GOLD[f"{f}/P{P}/x"]
    np.testing.assert_allclose(x.local_array.cpu().numpy(), gx, rtol=0, atol=xtol * np.abs(gx).max(),
                               err_msg=f"[rank {rank}] {f} x")

comm.Barrier()
torch.cuda.synchronize()
print(f"NSFILTERS_WORKER_OK rank={rank} size={P}")
