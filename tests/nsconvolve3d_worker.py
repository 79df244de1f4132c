"""NonStationaryConvolve3D at world size P under torchrun (one process per GPU): each rank's
MPIBlockDiag([NonStationaryConvolve3D] per volume) block against its volumes of the gathered reference fixtures of
tests/golden/nsconvolve3d_golden.npz, and the 3-D image-domain least-squares migration flow against its fixture.
Started by tests/test_nsconvolve3d.py."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import make_golden_nsconvolve3d as mg3  # noqa: E402
import pylops_mpi_b200 as pm  # noqa: E402

comm = pm.get_comm_world()
rank, P = comm.Get_rank(), comm.Get_size()
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "nsconvolve3d_golden.npz"), allow_pickle=False)


def block(nv_global, volume):
    """this rank's volumes of a (nv_global, ...) stack: (local_shapes, flat slice, first volume, volume count)"""
    rows = mg3.rows_of(P, nv_global)
    k0 = sum(rows[:rank])
    return [(r * volume,) for r in rows], slice(k0 * volume, (k0 + rows[rank]) * volume), k0, rows[rank]


def host(t):
    return t.cpu().numpy()


ls, sl, k0, nv = block(mg3.NV, mg3.NX * mg3.NY * mg3.NZ)
for nh, bank, dt in mg3.cases():
    hs, ih, x, v = mg3.case_inputs(nh, bank, dt)
    Op = pm.MPIBlockDiag([pm.local.NonStationaryConvolve3D((mg3.NX, mg3.NY, mg3.NZ), hs[k], *ih, dtype=hs.dtype)
                          for k in range(k0, k0 + nv)], dtype=dt)
    gy, gya = mg3.decode(GOLD, mg3.key(nh, bank), dt)
    name = f"{mg3.key(nh, bank)}/{dt}"
    np.testing.assert_array_equal(host((Op @ pm.DistributedArray.to_dist(x, local_shapes=ls)).local_array), gy[sl],
                                  err_msg=f"[rank {rank}] {name}/y")
    np.testing.assert_array_equal(host((Op.H @ pm.DistributedArray.to_dist(v, local_shapes=ls)).local_array),
                                  gya[sl], err_msg=f"[rank {rank}] {name}/ya")

ls, sl, k0, nv = block(mg3.FLOW_NV, mg3.FLOW_NY * mg3.FLOW_NX * mg3.FLOW_NZ)
Op = pm.MPIBlockDiag([pm.local.NonStationaryConvolve3D((mg3.FLOW_NY, mg3.FLOW_NX, mg3.FLOW_NZ), GOLD["flow/hs"],
                                                       mg3.FLOW_IHY, mg3.FLOW_IHX, mg3.FLOW_IHZ)] * nv)
mmig = GOLD["flow/mmig"]
d = pm.DistributedArray.to_dist(mmig, local_shapes=ls)
x0 = pm.DistributedArray.to_dist(np.zeros_like(mmig), local_shapes=ls)
x, _, iiter, _, _, cost = pm.cgls(Op, d, x0=x0, niter=mg3.FLOW_NITER, tol=0.0)
assert iiter == int(GOLD[f"flow/P{P}/iiter"])
floor = 10 * float(GOLD["flow/cond"]) * 2.0 ** -53       # as tests/test_nsconvolve3d.py's flow_tolerance()
xtol, ctol = (max(100 * float(s), floor) for s in GOLD["flow/spread"])
np.testing.assert_allclose(np.asarray(cost), GOLD[f"flow/P{P}/cost"], rtol=ctol, err_msg=f"[rank {rank}] cost")
gx = GOLD[f"flow/P{P}/x"]
np.testing.assert_allclose(host(x.local_array), gx[sl], rtol=0, atol=xtol * np.abs(gx).max(),
                           err_msg=f"[rank {rank}] x")

comm.Barrier()
torch.cuda.synchronize()
print(f"NSCONVOLVE3D_WORKER_OK rank={rank} size={P}")
