"""Restatement of third-party ``pylops.signalprocessing.Sliding1D`` (pylops 2.x, as remembered: pylops is not
installed here to check it) -- TEST INFRASTRUCTURE for tests/golden/make_golden_patch.py.  Windows of ``nwin``
samples of a 1-D signal of ``dimd`` samples start every ``nwin - nover`` samples; the model is ``nwins * nop``, window
``w``'s block contiguous.  pylops' chain ``HStack([Restriction.H]) * BlockDiag([Diagonal(tap_w) * Op])`` is
patch2d's ``_Patches`` with one window axis.

Remembered items: ``sliding1d_design`` and its return; the ``ValueError`` of a model ``dim`` other than
``nwins * Op.shape[1]`` (and, restated here, of an ``Op`` whose data are not ``nwin`` samples); the tapers
``taper(nwin, nover, tapertype)`` with the first window's leading ``nover`` samples and the last window's trailing
``nover`` set to 1, assigned in that order (one window: the trailing ones only)."""
import numpy as np

from ..utils.tapers import taper
from .patch2d import _Patches
from .sliding2d import _slidingsteps


def sliding1d_design(dimd, nwin, nover, nop):
    """(nwins, dim, mwin_inends, dwin_inends) of a Sliding1D on ``dimd`` samples with inner model ``nop``"""
    dwin_ins, dwin_ends = _slidingsteps(dimd, nwin, nover)
    nwins = len(dwin_ins)
    dim = nwins * nop
    mwin_ins, mwin_ends = _slidingsteps(dim, nop, 0)
    return nwins, dim, (mwin_ins, mwin_ends), (dwin_ins, dwin_ends)


def window_tapers(nwins, nwin, nover, tapertype):
    if tapertype is None:
        return None
    tap = taper(nwin, nover, tapertype)
    tapin, tapend = tap.copy(), tap.copy()
    tapin[:nover] = 1
    tapend[-nover:] = 1
    taps = {0: tapin}
    for i in range(1, nwins - 1):
        taps[i] = tap
    taps[nwins - 1] = tapend
    return [taps[i] for i in range(nwins)]


class Sliding1D(_Patches):
    """Sliding1D(Op, dim, dimd, nwin, nover, tapertype="hanning", name="S")"""

    def __init__(self, Op, dim, dimd, nwin, nover, tapertype="hanning", name="S"):
        dim, dimd, nwin, nover = (int(np.prod(dim)), int(np.prod(dimd)), int(nwin), int(nover))
        starts, _ = _slidingsteps(dimd, nwin, nover)
        if len(starts) * Op.shape[1] != dim:
            raise ValueError(f"Model shape (dim={dim}) is not consistent with chosen number of windows. Run "
                             f"sliding1d_design to identify the correct number of windows for the current model size...")
        if Op.shape[0] != nwin:
            raise ValueError(f"Op has {Op.shape[0]} data values, a window {nwin}")
        self.nwin, self.nover, self.tapertype = nwin, nover, tapertype
        self._finish(Op, (dim,), (dimd,), (nwin,), [starts], window_tapers(len(starts), nwin, nover, tapertype),
                     name)
