"""Generate the 3-D Kirchhoff demigration fixtures by running the REAL reference's MPIVStack and cgls (a pylops-mpi
checkout named by PYLOPS_MPI_REFERENCE, imported unmodified through make_golden.load_reference) over refshim's
restated ``pylops.waveeqprocessing.Kirchhoff`` / ``LSM`` with a ``y`` axis (refshim/pylops/waveeqprocessing/
kirchhoff3d.py; its ``traveltime_tables`` docstring says where the 3-D addition order comes from).

    PYLOPS_MPI_REFERENCE=<checkout> python tests/golden/make_golden_kirchhoff3d.py   # writes kirchhoff3d_golden.npz

Operator cases, float64.  A (OP_NY, OP_NX, OP_NZ) image (ni = 210, not a multiple of 32), an OP_NRY x OP_NRX grid of
receivers at the surface and OP_NS sources per rank at P in {1, 2, 3}, with OP_NT samples: short enough that pairs
land past the record and exactly on nt - 2 / nt - 1 (checked here), and with sources on grid points (trav_srcs = 0
there).  The reflectivity is BROADCAST and the data SCATTERed by source.  Wavelets as in make_golden_kirchhoff.py:
[1.0] at offset 0, a 21-tap Ricker at its centre, and an asymmetric 5-tap wavelet at offsets 0 and 4.

  op/P{P}/{wav}/y    gathered forward VStack @ m     (m: ``op_inputs``)
  op/P{P}/{wav}/ya   adjoint VStack.H @ d           (d: ``op_inputs``, the gathered data of P ranks)

Flow: 3-D least-squares migration (``flow_setup``: a (FLOW_NY, FLOW_NX, FLOW_NZ) image with two flat reflectors, a
3 x 3 receiver grid, FLOW_NS sources per rank, a 21-tap Ricker, FLOW_NITER iterations of cgls with its default tol)
at P in {1, 2, 3}:

  flow/P{P}/{madj,minv,iiter,cost}   VStack.H @ (VStack @ refl), and cgls's model, iterations and cost history
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden_kirchhoff import REFSHIM, WAVELETS, key, refshim, wavelet  # noqa: E402,F401

OP_NY, OP_NX, OP_NZ, OP_NRY, OP_NRX, OP_NS, OP_NT, OP_D, OP_DT, OP_VEL = 5, 7, 6, 3, 2, 2, 14, 4.0, 0.004, 1000.0
OP_NR = OP_NRY * OP_NRX
FLOW_NY, FLOW_NX, FLOW_NZ, FLOW_NS, FLOW_NT, FLOW_NITER = 9, 11, 12, 2, 60, 30
FLOW_NR = 9


def refshim3d():
    """refshim's 3-D restatement, ``pylops.waveeqprocessing.kirchhoff3d`` (refshim/ is on the path only while it is
    imported)"""
    added = REFSHIM not in sys.path
    if added:
        sys.path.insert(0, REFSHIM)
    try:
        import pylops.waveeqprocessing.kirchhoff3d as kirchhoff3d
    finally:
        if added:
            sys.path.remove(REFSHIM)
    return kirchhoff3d


def op_geometry(P, rank=None):
    """z, x, t, srcs (of ``rank``, or of all P ranks; rows (y, x, z)), recs, vel, y of the operator cases"""
    y, x, z = np.arange(OP_NY) * OP_D, np.arange(OP_NX) * OP_D, np.arange(OP_NZ) * OP_D
    t = np.arange(OP_NT) * OP_DT
    RY, RX = np.meshgrid(np.linspace(OP_D, (OP_NY - 2) * OP_D, OP_NRY), np.linspace(OP_D, (OP_NX - 2) * OP_D, OP_NRX),
                         indexing="ij")
    recs = np.vstack((RY.ravel(), RX.ravel(), np.zeros(OP_NR)))
    nstot = OP_NS * P
    sytot = np.round(np.linspace(0, OP_NY - 1, nstot)) * OP_D            # on grid points: trav_srcs = 0 there
    sxtot = np.round(np.linspace(OP_NX - 1, 0, nstot)) * OP_D
    sztot = np.full(nstot, OP_D)
    srcs = np.vstack((sytot, sxtot, sztot))
    if rank is not None:
        srcs = srcs[:, rank * OP_NS:(rank + 1) * OP_NS]
    return z, x, t, srcs, recs, OP_VEL, y


def op_inputs(P):
    """the image m (BROADCAST) and the gathered data d (P * OP_NS * OP_NR * OP_NT, scattered by source)"""
    rng = np.random.default_rng(41 + P)
    return rng.standard_normal(OP_NY * OP_NX * OP_NZ), rng.standard_normal(P * OP_NS * OP_NR * OP_NT)


def flow_setup(P, rank=None):
    """the 3-D flow at world size P: (z, x, t, sources of ``rank`` or of all ranks, recs, v0, wav, wavc, refl, y)"""
    ricker = refshim()[1].ricker
    d = 4
    y, x, z = np.arange(FLOW_NY) * d, np.arange(FLOW_NX) * d, np.arange(FLOW_NZ) * d
    v0 = 1000
    refl = np.zeros((FLOW_NY, FLOW_NX, FLOW_NZ))
    refl[:, :, 6] = -1
    refl[:, :, 10] = 0.5
    RY, RX = np.meshgrid(np.linspace(2 * d, (FLOW_NY - 3) * d, 3), np.linspace(2 * d, (FLOW_NX - 3) * d, 3),
                         indexing="ij")
    recs = np.vstack((RY.ravel(), RX.ravel(), 8 * np.ones(FLOW_NR)))
    nstot = FLOW_NS * P
    sytot = np.linspace(d, (FLOW_NY - 2) * d, nstot)
    sxtot = np.linspace((FLOW_NX - 2) * d, d, nstot)
    sources = np.vstack((sytot, sxtot, 4 * np.ones(nstot)))
    if rank is not None:
        sources = sources[:, rank * FLOW_NS:(rank + 1) * FLOW_NS]
    dt = 0.004
    t = np.arange(FLOW_NT) * dt
    wav, wavt, wavc = ricker(t[:11], f0=30)
    return z, x, t, sources, recs, v0, wav, wavc, refl, y


def main():
    from make_golden import load_reference          # puts refshim/ (mpi4py, pylops) on the path
    from mpi4py import MPI
    from pylops.waveeqprocessing.kirchhoff3d import LSM, Kirchhoff, traveltime_tables
    pkg, mods = load_reference()
    import importlib
    basic = importlib.import_module("pylops_mpi.optimization.basic")
    DA, Partition = pkg.DistributedArray, pkg.Partition
    VS = mods["VStack"].MPIVStack
    out = {}

    # the operator cases must exercise the record's end and trav = 0
    z, x, t, srcs, recs, vel, y = op_geometry(3)
    ts, tr = traveltime_tables(z, x, srcs, recs, vel, y=y)
    q = np.trunc((ts[:, :, None] + tr[:, None, :]) / OP_DT)
    for v in (OP_NT - 2, OP_NT - 1):
        assert np.any(q == v), v
    assert np.any(q > OP_NT - 1) and np.any(ts == 0)

    def t_op(rank, P, name):
        z, x, t, srcs, recs, vel, y = op_geometry(P, rank)
        w, off = wavelet(name)
        m, d = op_inputs(P)
        Op = VS(ops=[Kirchhoff(z, x, t, srcs, recs, vel, w, off, y=y, mode="analytic")])
        m_dist = DA(global_shape=m.size, partition=Partition.BROADCAST)
        m_dist[:] = m
        n = OP_NS * OP_NR * OP_NT
        d_dist = DA(global_shape=d.size, local_shapes=[(n,)] * P)
        d_dist[:] = d[rank * n:(rank + 1) * n]
        return {"y": (Op @ m_dist).asarray(), "ya": (Op.H @ d_dist).asarray()}

    for P in (1, 2, 3):
        for name in WAVELETS:
            res = MPI.run_world(P, t_op, P, name)[0]
            out[f"{key(P, name)}/y"] = res["y"]
            out[f"{key(P, name)}/ya"] = res["ya"]

    def t_flow(rank, P):
        z, x, t, sources, recs, v0, wav, wavc, refl, y = flow_setup(P, rank)
        lsm = LSM(z, x, t, sources, recs, v0, wav, wavc, y=y, mode="analytic")
        VStack = VS(ops=[lsm.Demop, ])
        refl_dist = DA(global_shape=refl.size, partition=Partition.BROADCAST)
        refl_dist[:] = refl.flatten()
        d_dist = VStack @ refl_dist
        madj_dist = VStack.H @ d_dist
        x0 = DA(VStack.shape[1], partition=Partition.BROADCAST)
        x0[:] = 0
        minv_dist, istop, iiter, r1, r2, cost = basic.cgls(VStack, d_dist, x0=x0, niter=FLOW_NITER)
        return madj_dist.asarray(), minv_dist.asarray(), iiter, cost

    for P in (1, 2, 3):
        madj, minv, iiter, cost = MPI.run_world(P, t_flow, P)[0]
        out[f"flow/P{P}/madj"] = np.asarray(madj)
        out[f"flow/P{P}/minv"] = np.asarray(minv)
        out[f"flow/P{P}/iiter"] = np.asarray(iiter)
        out[f"flow/P{P}/cost"] = np.asarray(cost)

    path = os.path.join(HERE, os.environ.get("GOLDEN_OUT", "kirchhoff3d_golden.npz"))
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1e6:.3f} MB")


if __name__ == "__main__":
    main()
