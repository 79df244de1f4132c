"""Generate the Kirchhoff demigration fixtures by running the REAL reference's MPIVStack and cgls (a pylops-mpi
checkout named by PYLOPS_MPI_REFERENCE, imported unmodified through make_golden.load_reference) over refshim's
restated ``pylops.waveeqprocessing.Kirchhoff`` / ``LSM`` and ``pylops.utils.wavelets.ricker``
(refshim/pylops/waveeqprocessing, refshim/pylops/utils/wavelets.py).

    PYLOPS_MPI_REFERENCE=<checkout> python tests/golden/make_golden_kirchhoff.py   # writes tests/golden/kirchhoff_golden.npz

Operator cases, float64.  A (OP_NX, OP_NZ) image, OP_NR receivers and OP_NS sources per rank at P in {1, 2, 3}, with
OP_NT samples: short enough that pairs land past the record and exactly on nt - 2 / nt - 1 (checked here), and with
sources on grid points (trav_srcs = 0 there).  The reflectivity is BROADCAST and the data SCATTERed by source, as in
tutorials/lsm.py.  Wavelets (``wavelet``): [1.0] at offset 0 (the convolution is the identity: the case pins the
spreading / stacking stage alone), a 21-tap Ricker at its centre, and an asymmetric 5-tap wavelet at offsets 0 and 4.

  op/P{P}/{wav}/y    gathered forward VStack @ m     (m: ``op_inputs``)
  op/P{P}/{wav}/ya   adjoint VStack.H @ d           (d: ``op_inputs``, the gathered data of P ranks)

Flow: tutorials/lsm.py at its own geometry (81 x 60 image, nr = 11, FLOW_NS sources per rank, nt = 651,
``ricker(t[:41], f0=20)``, FLOW_NITER iterations of cgls with its default tol) at P in {1, 2, 3}:

  flow/P{P}/{madj,minv,iiter,cost}   VStack.H @ (VStack @ refl), and cgls's model, iterations and cost history

The data are too large to store; the tests recompute them with the restatement (``flow_setup``).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

OP_NX, OP_NZ, OP_NR, OP_NS, OP_NT, OP_D, OP_DT, OP_VEL = 13, 9, 5, 2, 14, 4.0, 0.004, 1000.0
FLOW_NX, FLOW_NZ, FLOW_NR, FLOW_NS, FLOW_NT, FLOW_NITER = 81, 60, 11, 10, 651, 100
WAVELETS = ("spike", "ricker21", "asym/o0", "asym/o4")
REFSHIM = os.path.join(HERE, "refshim")


def refshim():
    """refshim's restated ``pylops.waveeqprocessing.kirchhoff`` and ``pylops.utils.wavelets`` modules (refshim/ is
    on the path only while they are imported)"""
    added = REFSHIM not in sys.path
    if added:
        sys.path.insert(0, REFSHIM)
    try:
        import pylops.utils.wavelets as wavelets
        import pylops.waveeqprocessing.kirchhoff as kirchhoff
    finally:
        if added:
            sys.path.remove(REFSHIM)
    return kirchhoff, wavelets


def key(P, wav):
    return f"op/P{P}/{wav}"


def wavelet(name):
    """(taps, offset) of an operator case"""
    if name == "spike":
        return np.array([1.0]), 0
    if name == "ricker21":
        w, _, wc = refshim()[1].ricker(np.arange(11) * OP_DT, f0=30)
        return w, int(wc)
    return np.array([1.0, -0.5, 0.25, 0.8, -0.3]), int(name[-1])


def op_geometry(P, rank=None):
    """z, x, t, srcs (of ``rank``, or of all P ranks), recs, vel of the operator cases"""
    x, z = np.arange(OP_NX) * OP_D, np.arange(OP_NZ) * OP_D
    t = np.arange(OP_NT) * OP_DT
    recs = np.vstack((np.linspace(2 * OP_D, (OP_NX - 3) * OP_D, OP_NR), np.zeros(OP_NR)))
    nstot = OP_NS * P
    sxtot = np.round(np.linspace(0, OP_NX - 1, nstot)) * OP_D            # on grid points: trav_srcs = 0 there
    sztot = np.full(nstot, OP_D)
    if rank is not None:
        sxtot, sztot = sxtot[rank * OP_NS:(rank + 1) * OP_NS], sztot[rank * OP_NS:(rank + 1) * OP_NS]
    return z, x, t, np.vstack((sxtot, sztot)), recs, OP_VEL


def op_inputs(P):
    """the image m (BROADCAST) and the gathered data d (P * OP_NS * OP_NR * OP_NT, scattered by source)"""
    rng = np.random.default_rng(31 + P)
    return rng.standard_normal(OP_NX * OP_NZ), rng.standard_normal(P * OP_NS * OP_NR * OP_NT)


def flow_setup(P, rank=None):
    """tutorials/lsm.py's geometry, wavelet and reflectivity at world size P: (z, x, t, sources of ``rank`` or of
    all ranks, recs, v0, wav, wavc, refl)"""
    ricker = refshim()[1].ricker
    nx, nz = FLOW_NX, FLOW_NZ
    dx, dz = 4, 4
    x, z = np.arange(nx) * dx, np.arange(nz) * dz
    v0 = 1000
    refl = np.zeros((nx, nz))
    refl[:, 30] = -1
    refl[:, 50] = 0.5
    nr = FLOW_NR
    rx = np.linspace(10 * dx, (nx - 10) * dx, nr)
    rz = 20 * np.ones(nr)
    recs = np.vstack((rx, rz))
    ns = FLOW_NS
    nstot = ns * P
    sxtot = np.linspace(dx * 10, (nx - 10) * dx, nstot)
    sztot = 10 * np.ones(nstot)
    if rank is None:
        sources = np.vstack((sxtot, sztot))
    else:
        sources = np.vstack((sxtot[rank * ns: (rank + 1) * ns], 10 * np.ones(ns)))
    nt = FLOW_NT
    dt = 0.004
    t = np.arange(nt) * dt
    wav, wavt, wavc = ricker(t[:41], f0=20)
    return z, x, t, sources, recs, v0, wav, wavc, refl


def main():
    from make_golden import load_reference          # puts refshim/ (mpi4py, pylops) on the path
    from mpi4py import MPI
    from pylops.waveeqprocessing.kirchhoff import Kirchhoff, traveltime_tables
    from pylops.waveeqprocessing.lsm import LSM
    pkg, mods = load_reference()
    import importlib
    basic = importlib.import_module("pylops_mpi.optimization.basic")
    DA, Partition = pkg.DistributedArray, pkg.Partition
    VS = mods["VStack"].MPIVStack
    out = {}

    # the operator cases must exercise the record's end and trav = 0
    z, x, t, srcs, recs, vel = op_geometry(3)
    ts, tr = traveltime_tables(z, x, srcs, recs, vel)
    q = np.trunc((ts[:, :, None] + tr[:, None, :]) / OP_DT)
    for v in (OP_NT - 2, OP_NT - 1):
        assert np.any(q == v), v
    assert np.any(q > OP_NT - 1) and np.any(ts == 0)

    def t_op(rank, P, name):
        z, x, t, srcs, recs, vel = op_geometry(P, rank)
        w, off = wavelet(name)
        m, d = op_inputs(P)
        Op = VS(ops=[Kirchhoff(z, x, t, srcs, recs, vel, w, off, mode="analytic")])
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
        """tutorials/lsm.py, statement by statement"""
        z, x, t, sources, recs, v0, wav, wavc, refl = flow_setup(P, rank)
        lsm = LSM(z, x, t, sources, recs, v0, wav, wavc, mode="analytic", engine="numba")
        VStack = VS(ops=[lsm.Demop, ])
        refl_dist = DA(global_shape=FLOW_NX * FLOW_NZ, partition=Partition.BROADCAST)
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

    path = os.path.join(HERE, os.environ.get("GOLDEN_OUT", "kirchhoff_golden.npz"))
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1e6:.3f} MB")


if __name__ == "__main__":
    main()
