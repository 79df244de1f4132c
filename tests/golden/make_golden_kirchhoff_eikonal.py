"""Generate the eikonal Kirchhoff demigration fixtures by running the REAL reference's MPIVStack and cgls (a pylops-mpi
checkout named by PYLOPS_MPI_REFERENCE, imported unmodified through make_golden.load_reference) over refshim's
restated ``pylops.waveeqprocessing.Kirchhoff`` / ``LSM`` with ``mode="eikonal"``
(refshim/pylops/waveeqprocessing/kirchhoff_eikonal.py; its tables come from refshim's Jacobi eikonal solver,
eikonal.py, standing in for scikit-fmm).

    PYLOPS_MPI_REFERENCE=<checkout> python tests/golden/make_golden_kirchhoff_eikonal.py   # writes the .npz
    PYLOPS_MPI_REFERENCE=<checkout> python tests/golden/make_golden_kirchhoff_eikonal.py --reorder
        # reruns the flow with the spreading / stacking sums reordered and prints how far it moves

Operator cases, float64, 2-D (``op``) and 3-D (``op3``).  Velocity ``op_velocity``: a vertical gradient times a
slow lens, so rays bend and the solver needs more Jacobi steps than the grid's Manhattan extent (checked here).
Spacings are unequal.  Sources sit on corners and edges, off grid nodes, and one exactly half-way between two
nodes along z (snapped half to even); receivers are off-grid.  OP_NT / OP3_NT are short enough that pairs land past
the record and exactly on nt - 2 / nt - 1 (checked here).  P in {1, 2, 3}, the four wavelets of
make_golden_kirchhoff.py, BROADCAST reflectivity and data SCATTERed by source:

  op/P{P}/{wav}/{y,ya}, op3/P{P}/{wav}/{y,ya}    forward VStack @ m and adjoint VStack.H @ d (``op_inputs``)

Flow: tutorials/lsm.py with a velocity gradient FLOW_KV (``vel = outer(ones(nx), v0 + kv * z)``) and
``mode="eikonal"``, FLOW_NITER iterations of cgls with its default tol, at P in {1, 2, 3}:

  flow/P{P}/{madj,minv,iiter,cost}

No pair's ``trav / dt`` lies within DT_MARGIN of an integer (checked here), so no fixture hinges on the last bit of
a traveltime sum.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden_kirchhoff import REFSHIM, WAVELETS, refshim, wavelet  # noqa: E402,F401
import make_golden_kirchhoff as mgk  # noqa: E402

OP_NX, OP_NZ, OP_DX, OP_DZ, OP_NR, OP_NS, OP_NT, OP_DT = 13, 9, 4.0, 3.0, 5, 2, 17, 0.0037
OP3_NY, OP3_NX, OP3_NZ, OP3_D, OP3_NRY, OP3_NRX, OP3_NS, OP3_NT = 5, 7, 6, (3.0, 4.0, 2.5), 3, 2, 2, 11
FLOW_KV, FLOW_NITER = 1.37, 100
DT_MARGIN = 1e-9


def refshim_eikonal():
    """refshim's ``pylops.waveeqprocessing.kirchhoff_eikonal`` and ``eikonal`` modules (refshim/ is on the path only
    while they are imported)"""
    added = REFSHIM not in sys.path
    if added:
        sys.path.insert(0, REFSHIM)
    try:
        import pylops.waveeqprocessing.eikonal as eikonal
        import pylops.waveeqprocessing.kirchhoff_eikonal as kirchhoff_eikonal
    finally:
        if added:
            sys.path.remove(REFSHIM)
    return kirchhoff_eikonal, eikonal


def op_velocity(axes):
    """v = 900 + 30 * z (m/s, z in m) times a lens 45 % slower at its centre, on the grid of ``axes`` ((y,) x, z)"""
    grids = np.meshgrid(*axes, indexing="ij")
    z = grids[-1]
    centre = [0.5 * (a[0] + a[-1]) for a in axes]
    r2 = sum((g - c) ** 2 for g, c in zip(grids, centre))
    width2 = (0.25 * (axes[-2][-1] - axes[-2][0])) ** 2
    return (900.0 + 30.0 * z) * (1.0 - 0.45 * np.exp(-r2 / width2))


def op_geometry(P, rank=None):
    """2-D: z, x, t, srcs (of ``rank``, or of all P ranks), recs, vel"""
    x, z = np.arange(OP_NX) * OP_DX, np.arange(OP_NZ) * OP_DZ
    t = np.arange(OP_NT) * OP_DT
    recs = np.vstack((np.linspace(3.3, (OP_NX - 1) * OP_DX - 3.3, OP_NR), np.full(OP_NR, 1.2)))
    # corners, edges, off-grid points and z = 13.5 = 4.5 * dz: half-way, snapped to node 4 (half to even)
    sx = np.array([0.0, (OP_NX - 1) * OP_DX, 2.2, 25.1, 47.9, 10.3])
    sz = np.array([(OP_NZ - 1) * OP_DZ, 0.0, 13.5, 22.9, 11.0, 4.4])
    srcs = np.vstack((sx, sz))[:, :OP_NS * P]
    if rank is not None:
        srcs = srcs[:, rank * OP_NS:(rank + 1) * OP_NS]
    return z, x, t, srcs, recs, op_velocity((x, z))


def op3_geometry(P, rank=None):
    """3-D: z, x, t, srcs (rows (y, x, z)), recs, vel, y"""
    dy, dx, dz = OP3_D
    y, x, z = np.arange(OP3_NY) * dy, np.arange(OP3_NX) * dx, np.arange(OP3_NZ) * dz
    t = np.arange(OP3_NT) * OP_DT
    RY, RX = np.meshgrid(np.linspace(1.1, (OP3_NY - 1) * dy - 1.1, OP3_NRY),
                         np.linspace(1.3, (OP3_NX - 1) * dx - 1.3, OP3_NRX), indexing="ij")
    recs = np.vstack((RY.ravel(), RX.ravel(), np.full(OP3_NRY * OP3_NRX, 0.4)))
    sy = np.array([0.0, (OP3_NY - 1) * dy, 4.5, 7.1, 1.9, 12.0])       # 4.5 = 1.5 * dy: half-way, node 2
    sx = np.array([(OP3_NX - 1) * dx, 0.0, 11.2, 3.9, 24.0, 13.0])
    sz = np.array([(OP3_NZ - 1) * dz, (OP3_NZ - 1) * dz, 6.2, 3.75, 12.4, 8.1])     # 3.75 = 1.5 * dz: half-way, node 2
    srcs = np.vstack((sy, sx, sz))[:, :OP3_NS * P]
    if rank is not None:
        srcs = srcs[:, rank * OP3_NS:(rank + 1) * OP3_NS]
    return z, x, t, srcs, recs, op_velocity((y, x, z)), y


def op_inputs(P, three=False):
    """the image m (BROADCAST) and the gathered data d (scattered by source)"""
    rng = np.random.default_rng((61 if three else 51) + P)
    ni = OP3_NY * OP3_NX * OP3_NZ if three else OP_NX * OP_NZ
    n = (OP3_NS * OP3_NRY * OP3_NRX * OP3_NT) if three else (OP_NS * OP_NR * OP_NT)
    return rng.standard_normal(ni), rng.standard_normal(P * n)


def flow_setup(P, rank=None):
    """tutorials/lsm.py with ``kv = FLOW_KV``: (z, x, t, sources, recs, vel, wav, wavc, refl)"""
    z, x, t, sources, recs, v0, wav, wavc, refl = mgk.flow_setup(P, rank)
    vel = np.outer(np.ones(x.size), v0 + FLOW_KV * z)
    return z, x, t, sources, recs, vel, wav, wavc, refl


def check_geometry(ts, tr, dt, nt=None):
    """no trav / dt within DT_MARGIN of an integer; with nt: pairs on nt - 2, nt - 1 and past the record"""
    q = (ts[:, :, None] + tr[:, None, :]) / dt
    assert np.min(np.abs(q - np.round(q))) > DT_MARGIN, np.min(np.abs(q - np.round(q)))
    if nt is not None:
        tq = np.trunc(q)
        for v in (nt - 2, nt - 1):
            assert np.any(tq == v), v
        assert np.any(tq > nt - 1)


def check_cases():
    """the geometry assertions of the module docstring, for every table the fixtures use"""
    KE, ek = refshim_eikonal()
    z, x, t, srcs, recs, vel = op_geometry(3)
    check_geometry(*KE.traveltime_tables(z, x, srcs, recs, vel), OP_DT, OP_NT)
    _, iters = ek.jacobi(vel[None], ek.spacings((x, z)), ek.snap(srcs, (x, z)))
    assert iters > (OP_NX - 1) + (OP_NZ - 1), iters
    assert ek.snap(srcs, (x, z))[2, 2] == 4                            # half-way along z, half to even
    z, x, t, srcs, recs, vel, y = op3_geometry(3)
    check_geometry(*KE.traveltime_tables(z, x, srcs, recs, vel, y=y), OP_DT, OP3_NT)
    nodes = ek.snap(srcs, (y, x, z))
    _, iters = ek.jacobi(vel, ek.spacings((y, x, z)), nodes)
    assert iters > (OP3_NY - 1) + (OP3_NX - 1) + (OP3_NZ - 1), iters
    assert nodes[2, 0] == 2 and nodes[3, 2] == 2
    z, x, t, sources, recs, vel, *_ = flow_setup(3)
    check_geometry(*KE.traveltime_tables(z, x, sources, recs, vel), t[1] - t[0])


def main(reorder=False):
    from make_golden import load_reference          # puts refshim/ (mpi4py, pylops) on the path
    from mpi4py import MPI
    from pylops.waveeqprocessing import kirchhoff
    from pylops.waveeqprocessing.kirchhoff_eikonal import LSM, Kirchhoff
    pkg, mods = load_reference()
    import importlib
    basic = importlib.import_module("pylops_mpi.optimization.basic")
    DA, Partition = pkg.DistributedArray, pkg.Partition
    VS = mods["VStack"].MPIVStack
    check_cases()
    out = {}

    def t_op(rank, P, name, three):
        w, off = wavelet(name)
        m, d = op_inputs(P, three)
        if three:
            z, x, t, srcs, recs, vel, y = op3_geometry(P, rank)
            n = OP3_NS * OP3_NRY * OP3_NRX * OP3_NT
        else:
            (z, x, t, srcs, recs, vel), y = op_geometry(P, rank), None
            n = OP_NS * OP_NR * OP_NT
        Op = VS(ops=[Kirchhoff(z, x, t, srcs, recs, vel, w, off, y=y, mode="eikonal")])
        m_dist = DA(global_shape=m.size, partition=Partition.BROADCAST)
        m_dist[:] = m
        d_dist = DA(global_shape=d.size, local_shapes=[(n,)] * P)
        d_dist[:] = d[rank * n:(rank + 1) * n]
        return {"y": (Op @ m_dist).asarray(), "ya": (Op.H @ d_dist).asarray()}

    if not reorder:
        for three, tag in ((False, "op"), (True, "op3")):
            for P in (1, 2, 3):
                for name in WAVELETS:
                    res = MPI.run_world(P, t_op, P, name, three)[0]
                    out[f"{tag}/P{P}/{name}/y"] = res["y"]
                    out[f"{tag}/P{P}/{name}/ya"] = res["ya"]

    class Reordered(Kirchhoff):
        """the same operator with its sums reordered: spreading over image points descending (``order`` 1), and
        stacking over traces descending too (``order`` 2)"""
        order = 0

        def _matvec(self, x):
            if self.order < 1:
                return super()._matvec(x)
            y = kirchhoff.spread(np.asarray(x).ravel()[::-1], self.trav_srcs[::-1], self.trav_recs[::-1], self.dt,
                                 self.nt, self.dtype)
            return self.cop._matvec(y.ravel())

        def _rmatvec(self, x):
            if self.order < 2:
                return super()._rmatvec(x)
            x = self.cop._rmatvec(np.asarray(x).ravel()).reshape(self.ns, self.nr, self.nt)[::-1, ::-1]
            return kirchhoff.stack(x.ravel(), self.trav_srcs[:, ::-1], self.trav_recs[:, ::-1], self.dt, self.nt,
                                   self.dtype)

    def t_flow(rank, P, order):
        """tutorials/lsm.py, statement by statement, with kv != 0 and mode="eikonal" """
        z, x, t, sources, recs, vel, wav, wavc, refl = flow_setup(P, rank)
        lsm = LSM(z, x, t, sources, recs, vel, wav, wavc, mode="eikonal")
        if order:
            lsm.Demop.__class__ = Reordered
            lsm.Demop.order = order
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
        madj, minv, iiter, cost = MPI.run_world(P, t_flow, P, 0)[0]
        if reorder:
            for order in (1, 2):
                _, mr, ir, cr = MPI.run_world(P, t_flow, P, order)[0]
                n = min(len(cost), len(cr))
                print(f"P={P} order={order}: iiter {iiter} vs {ir}, cost rel "
                      f"{np.max(np.abs(np.asarray(cr[:n]) - cost[:n]) / np.abs(cost[:n])):.3e}, minv "
                      f"{np.max(np.abs(mr - minv)) / np.max(np.abs(minv)):.3e}")
            continue
        out[f"flow/P{P}/madj"] = np.asarray(madj)
        out[f"flow/P{P}/minv"] = np.asarray(minv)
        out[f"flow/P{P}/iiter"] = np.asarray(iiter)
        out[f"flow/P{P}/cost"] = np.asarray(cost)

    if reorder:
        return
    path = os.path.join(HERE, os.environ.get("GOLDEN_OUT", "kirchhoff_eikonal_golden.npz"))
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1e6:.3f} MB")


if __name__ == "__main__":
    main(reorder="--reorder" in sys.argv)
