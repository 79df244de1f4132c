"""Radon2D / Radon3D at world size P under torchrun (one process per GPU): each rank's MPIBlockDiag of its gathers
against its slice of the gathered reference fixtures of tests/golden/radon_golden.npz (the exact cases, bit for bit),
and the denoising FISTA flow against its fixture.  Started by tests/test_radon.py."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import make_golden_radon as mgr  # noqa: E402
import pylops_mpi_b200 as pm  # noqa: E402

comm = pm.get_comm_world()
rank, P = comm.Get_rank(), comm.Get_size()
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "radon_golden.npz"), allow_pickle=False)


def host(t):
    return t.cpu().numpy()


def split(n_per, ng=mgr.NG):
    """local shapes of ng gathers of n_per values over the ranks, and this rank's slice"""
    rows = mgr.rows_of(P, ng)
    lo, hi = sum(rows[:rank]) * n_per, sum(rows[:rank + 1]) * n_per
    return [(r * n_per,) for r in rows], slice(lo, hi), rows[rank]


for case in mgr.cases():
    ndim, kind, interp, centeredh, nh = case
    if not mgr.exact(kind, interp):
        continue
    nm, nd = mgr.sizes(ndim, kind, nh)
    lsm, slm, ng = split(nm)
    lsd, sld, _ = split(nd)
    cls = pm.local.Radon2D if ndim == 2 else pm.local.Radon3D
    for dt in mgr.DTYPES:
        if dt == "complex128" and not mgr.complex_case(kind, interp, centeredh):
            continue
        x, v = mgr.case_inputs(*case, dt)
        Op = pm.MPIBlockDiag([cls(mgr.taxis(ndim), *mgr.axes(ndim, kind, centeredh, nh), kind=kind,
                                  centeredh=centeredh, interp=interp, dtype="float32" if dt == "float32" else "float64")
                              for _ in range(ng)], dtype=dt)
        gy, gya = mgr.decode(GOLD, mgr.key(*case), dt)
        name = f"{mgr.key(*case)}/{dt}"
        np.testing.assert_array_equal(host((Op @ pm.DistributedArray.to_dist(x, local_shapes=lsm)).local_array),
                                      gy[sld], err_msg=f"[rank {rank}] {name}/y")
        np.testing.assert_array_equal(host((Op.H @ pm.DistributedArray.to_dist(v, local_shapes=lsd)).local_array),
                                      gya[slm], err_msg=f"[rank {rank}] {name}/ya")

t, h, p = mgr.flow_axes()
nd, nm = mgr.FLOW_NH * mgr.FLOW_NT, p.size * mgr.FLOW_NT
lsd, sld, ng = split(nd, mgr.FLOW_NG)
lsm, slm, _ = split(nm, mgr.FLOW_NG)
Op = pm.MPIBlockDiag([pm.local.Radon2D(t, h, p, kind="linear") for _ in range(ng)])
d = pm.DistributedArray.to_dist(GOLD["flow/d"], local_shapes=lsd)
x0 = pm.DistributedArray.to_dist(np.zeros(mgr.FLOW_NG * nm), local_shapes=lsm)
x, iiter, cost = pm.fista(Op, d, x0, niter=mgr.FLOW_NITER, eps=mgr.FLOW_EPS, alpha=float(GOLD["flow/alpha"]), tol=1e-10)
assert iiter == int(GOLD[f"flow/P{P}/iiter"])
floor = 10 * float(GOLD["flow/cond"]) * 2.0 ** -53
xtol, ctol = (max(100 * float(s), floor) for s in GOLD["flow/spread"])
np.testing.assert_allclose(np.asarray(cost), GOLD[f"flow/P{P}/cost"], rtol=ctol, err_msg=f"[rank {rank}] cost")
gx = GOLD[f"flow/P{P}/x"]
np.testing.assert_allclose(host(x.local_array), gx[slm], rtol=0, atol=xtol * np.abs(gx).max(),
                           err_msg=f"[rank {rank}] x")

comm.Barrier()
torch.cuda.synchronize()
print(f"RADON_WORKER_OK rank={rank} size={P}")
