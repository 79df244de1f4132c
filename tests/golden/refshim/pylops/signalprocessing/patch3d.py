"""Restatement of third-party ``pylops.signalprocessing.Patch3D`` (pylops 2.x, as remembered: pylops is not installed
here to check it) -- TEST INFRASTRUCTURE for tests/golden/make_golden_patch.py.  Patch2D's restatement (patch2d.py)
with three window axes on ``dimsd = (ny, nx, nt)``: patch ``w = (i0 * nwins1 + i1) * nwins2 + i2``, model
``(nwins0 * nop[0], nwins1 * nop[1], nwins2 * nop[2])`` stored window-major.  pylops' chain ``HStack_0 *
BlockDiag([HStack_1] * nwins0) * BlockDiag([HStack_2] * nwins0 * nwins1) * BlockDiag([Diagonal(tap_w) * Op])`` sums
each sample over i2 within a strip, over i1 within a slab, then over i0, all ascending.

Remembered items (the least certain of this family): the base taper ``taper3d(nwin[2], nwin[:2], nover[:2],
tapertype)`` -- tapered along y and x, constant along t -- with Patch2D's edge rule on the (y, x) grid and the same
rule along t (the edge patches' outer ``nover[2]`` samples replaced by the middle sample, a no-op on a taper constant
along t); ``patch3d_design``; the ``ValueError`` of a model ``dims`` other than the above."""
import numpy as np

from ..utils.tapers import taper3d
from .patch2d import _Patches, _design, check, edge_tapers
from .sliding2d import _slidingsteps


def patch3d_design(dimsd, nwin, nover, nop):
    """(nwins, dims, mwins_inends, dwins_inends) of a Patch3D on data ``dimsd`` with inner model ``nop``"""
    return _design(dimsd, nwin, nover, nop)


def window_tapers(nwins, nwin, nover, tapertype):
    """the per-patch tapers (None: no taper)"""
    if tapertype is None:
        return None
    yx = edge_tapers(taper3d(nwin[2], nwin[:2], nover[:2], tapertype=tapertype), nwins[0], nwins[1], nwin, nover)
    mid2 = nwin[2] // 2
    taps = []
    for w in range(nwins[0] * nwins[1]):
        for i2 in range(nwins[2]):
            t = yx[w].copy()
            if i2 == 0 and nwins[2] > 1:
                t[:, :, :nover[2]] = t[:, :, mid2:mid2 + 1]
            if i2 == nwins[2] - 1:
                t[:, :, -nover[2]:] = t[:, :, mid2:mid2 + 1]
            taps.append(t)
    return taps


class Patch3D(_Patches):
    """Patch3D(Op, dims, dimsd, nwin, nover, nop, tapertype="hanning", scalings=None, name="P")"""

    def __init__(self, Op, dims, dimsd, nwin, nover, nop, tapertype="hanning", scalings=None, name="P"):
        dims, dimsd = tuple(int(d) for d in dims), tuple(int(d) for d in dimsd)
        nwin, nover, nop = tuple(int(v) for v in nwin), tuple(int(v) for v in nover), tuple(int(v) for v in nop)
        if scalings is not None:
            raise NotImplementedError("scalings are not restated")
        s = [_slidingsteps(dimsd[a], nwin[a], nover[a])[0] for a in (0, 1, 2)]
        nwins = tuple(len(si) for si in s)
        check(Op, dims, nwins, nop, nwin, "patch3d_design")
        self.nwin, self.nover, self.nop, self.tapertype = nwin, nover, nop, tapertype
        self._finish(Op, dims, dimsd, nwin, s, window_tapers(nwins, nwin, nover, tapertype), name)
