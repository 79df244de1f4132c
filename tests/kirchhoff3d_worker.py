"""3-D Kirchhoff demigration at world size P under torchrun (one process per GPU): each rank's Kirchhoff inside
MPIVStack against the gathered reference fixtures of tests/golden/kirchhoff3d_golden.npz (operator cases and the 3-D
least-squares migration flow), resident and with the traveltime tables forced into chunks.  Started by
tests/test_kirchhoff3d.py."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import make_golden_kirchhoff as mgk  # noqa: E402
import make_golden_kirchhoff3d as m3  # noqa: E402
import pylops_mpi_b200 as pm  # noqa: E402

comm = pm.get_comm_world()
rank, P = comm.Get_rank(), comm.Get_size()
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "kirchhoff3d_golden.npz"), allow_pickle=False)
# five times the spread of reordered-sum reruns of the fixture solve (see tests/test_kirchhoff3d.py)
FLOW_COST_RTOL, FLOW_MINV_ATOL = 0.55, 2e-2
BUDGET = pm.local.KIRCHHOFF_TABLE_BYTES


def host(t):
    return t.cpu().numpy()


def close(name, got, ref, atol_rel):
    np.testing.assert_allclose(got, ref, rtol=0, atol=atol_rel * np.abs(ref).max(), err_msg=f"[rank {rank}] {name}")


n = m3.OP_NS * m3.OP_NR * m3.OP_NT
ls = [(n,)] * P
for budget in (BUDGET, (m3.OP_NS + m3.OP_NR) * 8 * 64):          # resident, then chunks of 64 image points
    pm.local.KIRCHHOFF_TABLE_BYTES = budget
    for wav in mgk.WAVELETS:
        h, off = mgk.wavelet(wav)
        z, x, t, srcs, recs, vel, y = m3.op_geometry(P, rank)
        K = pm.local.Kirchhoff(z, x, t, srcs, recs, vel, h, off, y=y, mode="analytic")
        assert K.chunked == (budget != BUDGET)
        Op = pm.MPIVStack([K])
        m, d = m3.op_inputs(P)
        yf = Op @ pm.DistributedArray.to_dist(m, partition=pm.Partition.BROADCAST)
        ya = Op.H @ pm.DistributedArray.to_dist(d, local_shapes=ls)
        k = mgk.key(P, wav)
        close(f"{k}/y", host(yf.local_array), GOLD[f"{k}/y"][rank * n:(rank + 1) * n], 1e-12)
        close(f"{k}/ya", host(ya.local_array), GOLD[f"{k}/ya"], 1e-12)
pm.local.KIRCHHOFF_TABLE_BYTES = BUDGET

z, x, t, srcs, recs, v0, wav, wavc, refl, y = m3.flow_setup(P, rank)
lsm = pm.local.LSM(z, x, t, srcs, recs, v0, wav, wavc, y=y, mode="analytic")
VStack = pm.MPIVStack(ops=[lsm.Demop, ])
refl_dist = pm.DistributedArray(global_shape=refl.size, partition=pm.Partition.BROADCAST)
refl_dist[:] = refl.flatten()
d_dist = VStack @ refl_dist
madj = VStack.H @ d_dist
x0 = pm.DistributedArray(VStack.shape[1], partition=pm.Partition.BROADCAST)
x0[:] = 0
minv, _, iiter, _, _, cost = pm.cgls(VStack, d_dist, x0=x0, niter=m3.FLOW_NITER)
g = f"flow/P{P}"
close(f"{g}/madj", host(madj.local_array), GOLD[f"{g}/madj"], 1e-12)
assert int(iiter) == int(GOLD[f"{g}/iiter"])
np.testing.assert_allclose(np.asarray(cost), GOLD[f"{g}/cost"], rtol=FLOW_COST_RTOL, err_msg=f"[rank {rank}] cost")
close(f"{g}/minv", host(minv.local_array), GOLD[f"{g}/minv"], FLOW_MINV_ATOL)

comm.Barrier()
torch.cuda.synchronize()
print(f"KIRCHHOFF3D_WORKER_OK rank={rank} size={P}")
