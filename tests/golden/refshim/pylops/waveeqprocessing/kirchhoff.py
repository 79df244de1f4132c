"""Restatement of third-party ``pylops.waveeqprocessing.Kirchhoff`` (pylops 2.x, mode="analytic", 2-D,
dynamic=False, wavfilter=False) -- TEST INFRASTRUCTURE so that the reference's MPIVStack and cgls can be run over the
rank-local demigration of tutorials/lsm.py by tests/golden/make_golden_kirchhoff.py.

As pylops computes it:
  - tables, float64: ``X, Z = meshgrid(x, z, indexing="ij")`` raveled (``ii = ix * nz + iz``),
    ``trav_srcs[ii, s] = sqrt((X - sx)**2 + (Z - sz)**2) / vel``, the same for the receivers;
  - per (ii, isrc, irec): ``trav = trav_srcs[ii, s] + trav_recs[ii, r]``, ``itrav = int(trav / dt)``,
    ``travd = trav / dt - itrav``, used only when ``0 <= itrav < nt - 1``;
  - forward: for each trace ``isr = isrc * nr + irec`` and ii ascending, ``y[isr, itrav] += x[ii] * (1 - travd)``
    then ``y[isr, itrav + 1] += x[ii] * travd``; then ``Convolve1D((ns * nr, nt), wav, offset=wavcenter, axis=1)``;
  - adjoint: the Convolve1D adjoint, then for each ii and (isrc, irec) ascending
    ``y[ii] += x[isr, itrav] * (1 - travd) + x[isr, itrav + 1] * travd``.
The loops are vectorised without changing any floating-point operation or its order: ``np.add.at`` applies its
updates one by one in index order (the forward's interleaved first / second taps), and the adjoint adds one
(isrc, irec) pair at a time to the whole image."""
import numpy as np

from .. import LinearOperator
from ..signalprocessing.convolve1d import Convolve1D


def traveltime_tables(z, x, srcs, recs, vel):
    """(trav_srcs (ni, ns), trav_recs (ni, nr)), float64"""
    X, Z = np.meshgrid(x, z, indexing="ij")
    X, Z = X.ravel(), Z.ravel()
    trav_srcs = np.sqrt((X[:, None] - srcs[0][None]) ** 2 + (Z[:, None] - srcs[1][None]) ** 2) / vel
    trav_recs = np.sqrt((X[:, None] - recs[0][None]) ** 2 + (Z[:, None] - recs[1][None]) ** 2) / vel
    return trav_srcs.astype(np.float64), trav_recs.astype(np.float64)


def pair_index(trav, dt, nt):
    """itrav (int64, 0 where unused), travd, and the mask of used pairs"""
    q = trav / dt
    tq = np.trunc(q)
    ok = (tq >= 0) & (tq < nt - 1)
    it = np.where(ok, tq, 0).astype(np.int64)
    return it, q - it, ok


def spread(x, trav_srcs, trav_recs, dt, nt, dtype):
    """the forward's spreading stage: (ns * nr, nt) traces of dtype"""
    ni, ns = trav_srcs.shape
    nr = trav_recs.shape[1]
    y = np.zeros((ns * nr, nt), dtype=dtype)
    trav = (trav_srcs[:, :, None] + trav_recs[:, None, :]).reshape(ni, ns * nr).T      # (isr, ii)
    it, d, ok = pair_index(trav, dt, nt)
    isr, ii = np.nonzero(ok)                                                             # (isr, ii) ascending
    base = isr * nt + it[isr, ii]
    xv = x[ii]
    idx = np.stack((base, base + 1), axis=1).ravel()                                     # first tap, then second
    val = np.stack((xv * (1 - d[isr, ii]), xv * d[isr, ii]), axis=1).ravel()
    np.add.at(y.reshape(-1), idx, val)
    return y


def stack(x, trav_srcs, trav_recs, dt, nt, dtype):
    """the adjoint's stacking stage: the (ni,) image of dtype from (ns * nr, nt) traces"""
    ni, ns = trav_srcs.shape
    nr = trav_recs.shape[1]
    y = np.zeros(ni, dtype=dtype)
    x = x.reshape(ns * nr, nt)
    for isrc in range(ns):
        for irec in range(nr):
            it, d, ok = pair_index(trav_srcs[:, isrc] + trav_recs[:, irec], dt, nt)
            xt = x[isrc * nr + irec]
            y[ok] += xt[it[ok]] * (1 - d[ok]) + xt[it[ok] + 1] * d[ok]
    return y


class Kirchhoff(LinearOperator):
    def __init__(self, z, x, t, srcs, recs, vel, wav, wavcenter, y=None, mode="eikonal", wavfilter=False,
                 dynamic=False, trav=None, amp=None, aperture=None, angleaperture=90, snell=None, engine="numpy",
                 dtype="float64", name="K"):
        if mode != "analytic" or y is not None or wavfilter or dynamic or trav is not None or amp is not None \
                or aperture is not None or angleaperture != 90 or snell is not None:
            raise NotImplementedError("only mode='analytic', 2-D, static, without filtering or apertures is restated")
        if not isinstance(vel, (float, int, np.floating, np.integer)):
            raise ValueError("vel must be scalar for mode=analytical")
        self.nx, self.nz, self.nt = len(x), len(z), len(t)
        self.ns, self.nr = srcs.shape[1], recs.shape[1]
        self.dt = t[1] - t[0]
        self.trav_srcs, self.trav_recs = traveltime_tables(z, x, srcs, recs, vel)
        self.cop = Convolve1D((self.ns * self.nr, self.nt), h=wav, offset=wavcenter, axis=1, dtype=dtype)
        self.dims, self.dimsd = (self.nx, self.nz), (self.ns, self.nr, self.nt)
        super().__init__(dtype=np.dtype(dtype), shape=(self.ns * self.nr * self.nt, self.nx * self.nz))

    def _matvec(self, x):
        y = spread(np.asarray(x).ravel(), self.trav_srcs, self.trav_recs, self.dt, self.nt, self.dtype)
        return self.cop._matvec(y.ravel())

    def _rmatvec(self, x):
        x = self.cop._rmatvec(np.asarray(x).ravel())
        return stack(x, self.trav_srcs, self.trav_recs, self.dt, self.nt, self.dtype)
