"""Restatement of third-party ``pylops.waveeqprocessing.Kirchhoff`` / ``LSM`` (pylops 2.x, mode="analytic",
dynamic=False, wavfilter=False) WITH a ``y`` axis -- TEST INFRASTRUCTURE so that the reference's MPIVStack and cgls
can be run over the 3-D rank-local demigration by tests/golden/make_golden_kirchhoff3d.py.

Only the traveltime tables and the image shape differ from 2-D: the spreading / stacking stages and the wavelet
convolution are the 2-D restatement's own (``kirchhoff.spread`` / ``kirchhoff.stack``, ``Convolve1D``), and without
``y`` everything here is the 2-D restatement unchanged (``kirchhoff.traveltime_tables``)."""
import numpy as np

from .. import LinearOperator
from ..signalprocessing.convolve1d import Convolve1D
from . import kirchhoff


def traveltime_tables(z, x, srcs, recs, vel, y=None):
    """(trav_srcs (ni, ns), trav_recs (ni, nr)), float64; the 2-D restatement's tables when ``y`` is None.

    3-D: the grid is ``Y, X, Z = meshgrid(y, x, z, indexing="ij")`` raveled (``ii = (iy * nx + ix) * nz + iz``),
    ``srcs`` / ``recs`` have rows ``(y, x, z)``, and ``dist2 = (X - sx)**2 + (Z - sz)**2``, then
    ``dist2 += (Y - sy)**2``, then ``trav = sqrt(dist2) / vel``.  That addition order is pylops 2.x's
    ``Kirchhoff._traveltime_table`` as remembered, not checked against its source (pylops is not available here):
    fixtures made from this restatement are bit-exact to it, and would differ from pylops by at most about one ulp of
    traveltime if pylops adds the three terms in another order."""
    if y is None:
        return kirchhoff.traveltime_tables(z, x, srcs, recs, vel)
    Y, X, Z = np.meshgrid(y, x, z, indexing="ij")
    Y, X, Z = Y.ravel(), X.ravel(), Z.ravel()

    def table(pts):
        dist2 = (X[:, None] - pts[1][None]) ** 2 + (Z[:, None] - pts[2][None]) ** 2
        dist2 += (Y[:, None] - pts[0][None]) ** 2
        return (np.sqrt(dist2) / vel).astype(np.float64)

    return table(srcs), table(recs)


class Kirchhoff(LinearOperator):
    def __init__(self, z, x, t, srcs, recs, vel, wav, wavcenter, y=None, mode="eikonal", wavfilter=False,
                 dynamic=False, trav=None, amp=None, aperture=None, angleaperture=90, snell=None, engine="numpy",
                 dtype="float64", name="K"):
        if mode != "analytic" or wavfilter or dynamic or trav is not None or amp is not None \
                or aperture is not None or angleaperture != 90 or snell is not None:
            raise NotImplementedError("only mode='analytic', static, without filtering or apertures is restated")
        if not isinstance(vel, (float, int, np.floating, np.integer)):
            raise ValueError("vel must be scalar for mode=analytical")
        self.nx, self.nz, self.nt = len(x), len(z), len(t)
        self.ns, self.nr = srcs.shape[1], recs.shape[1]
        self.dt = t[1] - t[0]
        self.trav_srcs, self.trav_recs = traveltime_tables(z, x, srcs, recs, vel, y=y)
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
    """pylops.waveeqprocessing.LSM for kind="kirchhoff": only ``Demop``, passing ``y`` through"""

    def __init__(self, z, x, t, srcs, recs, vel, wav, wavcenter, y=None, kind="kirchhoff", dottest=False,
                 **kwargs_mod):
        if kind != "kirchhoff" or dottest:
            raise NotImplementedError("only kind='kirchhoff' without dottest is restated")
        self.y, self.x, self.z, self.t = y, x, z, t
        self.Demop = Kirchhoff(z, x, t, srcs, recs, vel, wav, wavcenter, y=y, **kwargs_mod)
