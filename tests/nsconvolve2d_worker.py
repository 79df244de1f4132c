"""NonStationaryConvolve2D at world size P under torchrun (one process per GPU): each rank's
MPIBlockDiag([NonStationaryConvolve2D] per slice) block against its slice of the gathered reference fixtures of
tests/golden/nsconvolve2d_golden.npz, and the image-domain least-squares migration flow against its fixture.  Started
by tests/test_nsconvolve2d.py."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import make_golden_nsconvolve2d as mg2  # noqa: E402
import pylops_mpi_b200 as pm  # noqa: E402

comm = pm.get_comm_world()
rank, P = comm.Get_rank(), comm.Get_size()
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "nsconvolve2d_golden.npz"), allow_pickle=False)


def block(ny_global, plane):
    """this rank's slices of a (ny_global, ...) stack: (local_shapes, flat slice, first slice, slice count)"""
    rows = mg2.rows_of(P, ny_global)
    k0 = sum(rows[:rank])
    return [(r * plane,) for r in rows], slice(k0 * plane, (k0 + rows[rank]) * plane), k0, rows[rank]


def host(t):
    return t.cpu().numpy()


ls, sl, k0, ny = block(mg2.NY, mg2.NX * mg2.NZ)
for nh, bank, dt in mg2.cases():
    hs, ihx, ihz, x, v = mg2.case_inputs(nh, bank, dt)
    Op = pm.MPIBlockDiag([pm.local.NonStationaryConvolve2D((mg2.NX, mg2.NZ), hs[k], ihx, ihz, dtype=hs.dtype)
                          for k in range(k0, k0 + ny)], dtype=dt)
    gy, gya = mg2.decode(GOLD, mg2.key(nh, bank), dt)
    name = f"{mg2.key(nh, bank)}/{dt}"
    np.testing.assert_array_equal(host((Op @ pm.DistributedArray.to_dist(x, local_shapes=ls)).local_array), gy[sl],
                                  err_msg=f"[rank {rank}] {name}/y")
    np.testing.assert_array_equal(host((Op.H @ pm.DistributedArray.to_dist(v, local_shapes=ls)).local_array),
                                  gya[sl], err_msg=f"[rank {rank}] {name}/ya")

ls, sl, k0, ny = block(mg2.FLOW_NY, mg2.FLOW_NX * mg2.FLOW_NZ)
Op = pm.MPIBlockDiag([pm.local.NonStationaryConvolve2D((mg2.FLOW_NX, mg2.FLOW_NZ), GOLD["flow/hs"], mg2.FLOW_IHX,
                                                       mg2.FLOW_IHZ)] * ny)
mmig = GOLD["flow/mmig"]
d = pm.DistributedArray.to_dist(mmig, local_shapes=ls)
x0 = pm.DistributedArray.to_dist(np.zeros_like(mmig), local_shapes=ls)
x, _, iiter, _, _, cost = pm.cgls(Op, d, x0=x0, niter=mg2.FLOW_NITER, tol=0.0)
assert iiter == int(GOLD[f"flow/P{P}/iiter"])
np.testing.assert_allclose(np.asarray(cost), GOLD[f"flow/P{P}/cost"], rtol=1e-10, err_msg=f"[rank {rank}] cost")
gx = GOLD[f"flow/P{P}/x"]
np.testing.assert_allclose(host(x.local_array), gx[sl], rtol=1e-9, atol=1e-10 * np.abs(gx).max(),
                           err_msg=f"[rank {rank}] x")

comm.Barrier()
torch.cuda.synchronize()
print(f"NSCONVOLVE2D_WORKER_OK rank={rank} size={P}")
