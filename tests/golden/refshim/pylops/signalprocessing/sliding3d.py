"""Restatement of third-party ``pylops.signalprocessing.Sliding3D`` (pylops 2.x, as remembered: pylops is not
installed here to check it) -- TEST INFRASTRUCTURE for tests/golden/make_golden_sliding.py.  Sliding2D's restatement
(sliding2d.py) with windows on the grid of axes 0 and 1 of ``dimsd = (n0, n1, nt)``: window ``w = i0 * nwins1 + i1``,
model ``(nwins0 * nop[0], nwins1 * nop[1], nop[2])`` stored window-major, as BlockDiag orders its blocks (block ``w``
of ``prod(nop)`` values contiguous).  pylops' chain ``HStack_0 * BlockDiag([HStack_1] * nwins0) * BlockDiag([Diagonal
(tap_w) * Op])`` sums each trace over i1 ascending within a row of windows, then over i0 ascending.

Remembered items: the ``ValueError`` of a model ``dims`` other than ``(nwins0 * nop[0], nwins1 * nop[1], nop[2])``;
the tapers ``taper3d(nt, nwin, nover, tapertype)``, with every edge window's outer ``nover`` rows (axis 0) or columns
(axis 1) replaced by the taper's middle row ``nwin[0] // 2`` / column ``nwin[1] // 2``, assigned in pylops' order --
top, bottom, left, right, then the four corners -- so that one window along an axis keeps only its trailing edge
replaced, as in 2-D.  ``nproc`` is accepted and ignored."""
import numpy as np

from ..utils.tapers import taper3d
from .sliding2d import _Sliding, _slidingsteps


def sliding3d_design(dimsd, nwin, nover, nop):
    """(nwins, dims, mwins_inends, dwins_inends) of a Sliding3D on data ``dimsd`` with inner model ``nop``"""
    d0 = _slidingsteps(dimsd[0], nwin[0], nover[0])
    d1 = _slidingsteps(dimsd[1], nwin[1], nover[1])
    nwins = (len(d0[0]), len(d1[0]))
    dims = (nwins[0] * nop[0], nwins[1] * nop[1], nop[2])
    m0 = _slidingsteps(dims[0], nop[0], 0)
    m1 = _slidingsteps(dims[1], nop[1], 0)
    return nwins, dims, (m0, m1, (0, dims[2])), (d0, d1, (0, dimsd[2]))


def window_tapers(nwins0, nwins1, nt, nwin, nover, tapertype):
    if tapertype is None:
        return None
    nwins = nwins0 * nwins1
    tap = taper3d(nt, nwin, nover, tapertype=tapertype)
    taps = {itap: tap for itap in range(nwins)}
    mid0, mid1 = nwin[0] // 2, nwin[1] // 2

    def rows(t, lead):
        t = t.copy()
        if lead:
            t[:nover[0]] = t[mid0]
        else:
            t[-nover[0]:] = t[mid0]
        return t

    def cols(t, lead):
        t = t.copy()
        if lead:
            t[:, :nover[1]] = t[:, mid1][:, np.newaxis, :]
        else:
            t[:, -nover[1]:] = t[:, mid1][:, np.newaxis, :]
        return t

    for itap in range(0, nwins1):
        taps[itap] = rows(tap, True)
    for itap in range(nwins - nwins1, nwins):
        taps[itap] = rows(tap, False)
    for itap in range(0, nwins, nwins1):
        taps[itap] = cols(tap, True)
    for itap in range(nwins1 - 1, nwins, nwins1):
        taps[itap] = cols(tap, False)
    taps[0] = rows(cols(tap, True), True)
    taps[nwins1 - 1] = rows(cols(tap, False), True)
    taps[nwins - nwins1] = rows(cols(tap, True), False)
    taps[nwins - 1] = rows(cols(tap, False), False)
    return [taps[i] for i in range(nwins)]


class Sliding3D(_Sliding):
    """Sliding3D(Op, dims, dimsd, nwin, nover, nop, tapertype="hanning", nproc=1, name="P")"""

    def __init__(self, Op, dims, dimsd, nwin, nover, nop, tapertype="hanning", nproc=1, name="P"):
        dims, dimsd = tuple(int(d) for d in dims), tuple(int(d) for d in dimsd)
        nwin, nover, nop = tuple(int(v) for v in nwin), tuple(int(v) for v in nover), tuple(int(v) for v in nop)
        s0, _ = _slidingsteps(dimsd[0], nwin[0], nover[0])
        s1, _ = _slidingsteps(dimsd[1], nwin[1], nover[1])
        if len(s0) * nop[0] != dims[0] or len(s1) * nop[1] != dims[1] or nop[2] != dims[2]:
            raise ValueError(f"Model shape (dims={dims}) is not consistent with chosen number of windows. Run "
                             f"sliding3d_design to identify the correct number of windows for the current model size...")
        if Op.shape[1] != int(np.prod(nop)):
            raise ValueError(f"Op has {Op.shape[1]} model values, nop {nop}")
        if Op.shape[0] != nwin[0] * nwin[1] * dimsd[2]:
            raise ValueError(f"Op has {Op.shape[0]} data values, a window {nwin[0]} x {nwin[1]} x {dimsd[2]}")
        self.dims, self.nwin, self.nover, self.nop, self.tapertype = dims, nwin, nover, nop, tapertype
        self.nproc = nproc
        self.dimsd3 = dimsd
        self._finish(Op, dimsd, (nwin[0], nwin[1], dimsd[2]), (s0, s1),
                     window_tapers(len(s0), len(s1), dimsd[2], nwin, nover, tapertype), name)
