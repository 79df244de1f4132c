"""Restatement of third-party ``pylops.waveeqprocessing.Kirchhoff`` / ``LSM`` (pylops 2.x, dynamic=False,
wavfilter=False) with ``mode="eikonal"`` and ``mode="byot"``, 2-D or, with ``y``, 3-D -- TEST INFRASTRUCTURE so that
the reference's MPIVStack and cgls can be run over the rank-local demigration in a velocity model by
tests/golden/make_golden_kirchhoff_eikonal.py.

Only the traveltime tables differ from the analytic restatements: the spreading / stacking stages and the wavelet
convolution are the 2-D restatement's own (``kirchhoff.spread`` / ``kirchhoff.stack``, ``Convolve1D``).

  - ``mode="eikonal"``: pylops 2.x's eikonal branch as remembered (pylops is not available here): each point is
    snapped to the node ``round((p - axis[0]) / d)`` per axis and its table is ``skfmm.travel_time`` through ``vel``,
    raveled as the analytic tables.  scikit-fmm is replaced by ``eikonal.traveltime_table``, a first-order Jacobi
    solver with T = 0 on the node (its docstring lists how that differs from scikit-fmm).
  - ``mode="byot"``: ``trav=(trav_srcs, trav_recs)`` of shapes (ni, ns) / (ni, nr), used as given (float64).
  - ``mode="analytic"``: the analytic restatements, for comparison."""
import numpy as np

from .. import LinearOperator
from ..signalprocessing.convolve1d import Convolve1D
from . import eikonal, kirchhoff, kirchhoff3d


def traveltime_tables(z, x, srcs, recs, vel, y=None, mode="eikonal", trav=None):
    """(trav_srcs (ni, ns), trav_recs (ni, nr)), float64, of ``mode``"""
    if mode == "analytic":
        return kirchhoff3d.traveltime_tables(z, x, srcs, recs, vel, y=y)
    if mode == "byot":
        ts, tr = trav
        return np.asarray(ts, dtype=np.float64), np.asarray(tr, dtype=np.float64)
    if mode != "eikonal":
        raise NotImplementedError(mode)
    axes = (x, z) if y is None else (y, x, z)
    return eikonal.traveltime_table(vel, axes, srcs), eikonal.traveltime_table(vel, axes, recs)


class Kirchhoff(LinearOperator):
    def __init__(self, z, x, t, srcs, recs, vel, wav, wavcenter, y=None, mode="eikonal", wavfilter=False,
                 dynamic=False, trav=None, amp=None, aperture=None, angleaperture=90, snell=None, engine="numpy",
                 dtype="float64", name="K"):
        if wavfilter or dynamic or amp is not None or aperture is not None or angleaperture != 90 \
                or snell is not None:
            raise NotImplementedError("only the static operator without filtering or apertures is restated")
        self.nx, self.nz, self.nt = len(x), len(z), len(t)
        self.ns, self.nr = srcs.shape[1], recs.shape[1]
        self.dt = t[1] - t[0]
        self.trav_srcs, self.trav_recs = traveltime_tables(z, x, srcs, recs, vel, y=y, mode=mode, trav=trav)
        self.cop = Convolve1D((self.ns * self.nr, self.nt), h=wav, offset=wavcenter, axis=1, dtype=dtype)
        self.dims = (self.nx, self.nz) if y is None else (len(y), self.nx, self.nz)
        self.dimsd = (self.ns, self.nr, self.nt)
        super().__init__(dtype=np.dtype(dtype), shape=(self.ns * self.nr * self.nt, int(np.prod(self.dims))))

    def _matvec(self, x):
        y = kirchhoff.spread(np.asarray(x).ravel(), self.trav_srcs, self.trav_recs, self.dt, self.nt, self.dtype)
        return self.cop._matvec(y.ravel())

    def _rmatvec(self, x):
        x = self.cop._rmatvec(np.asarray(x).ravel())
        return kirchhoff.stack(x, self.trav_srcs, self.trav_recs, self.dt, self.nt, self.dtype)


class LSM:
    """pylops.waveeqprocessing.LSM for kind="kirchhoff": only ``Demop``, passing ``y`` and ``kwargs_mod`` through"""

    def __init__(self, z, x, t, srcs, recs, vel, wav, wavcenter, y=None, kind="kirchhoff", dottest=False,
                 **kwargs_mod):
        if kind != "kirchhoff" or dottest:
            raise NotImplementedError("only kind='kirchhoff' without dottest is restated")
        self.y, self.x, self.z, self.t = y, x, z, t
        self.Demop = Kirchhoff(z, x, t, srcs, recs, vel, wav, wavcenter, y=y, **kwargs_mod)
