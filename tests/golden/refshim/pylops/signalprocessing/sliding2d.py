"""Restatement of third-party ``pylops.signalprocessing.Sliding2D`` (pylops 2.x, as remembered: pylops is not
installed here to check it) -- TEST INFRASTRUCTURE so that the reference's MPIBlockDiag and FISTA can be run over
sliding-window operators by tests/golden/make_golden_sliding.py.

Windows of ``nwin`` traces run along axis 0 of the data ``dimsd = (n, nt)``, starting every ``nwin - nover`` traces
(``_slidingsteps``).  The model is ``(nwins * nop[0], nop[1])``, window ``w``'s block contiguous.  pylops builds
``HStack([Restriction.H]) * BlockDiag([Diagonal(tap_w) * Op])``; this restatement applies that chain in its order:

    y = 0;  for w ascending:  y[start_w:end_w] += tap_w * Op.matvec(x_w)         (tap_w of Op's dtype)
    x_w = Op.rmatvec(tap_w * d[start_w:end_w])

Remembered items: the steps ``arange(0, n - nwin + 1, nwin - nover)`` and the ``ValueError`` for ``nwin > n``; the
``ValueError`` of a model ``dims`` other than ``(nwins * nop[0], nop[1])`` (and, restated here, of ``nover >= nwin``
and of an ``Op`` whose data is not a ``(nwin, nt)`` window); the tapers ``taper2d(nt, nwin, nover, tapertype)`` with
the first window's leading ``nover`` samples and the last window's trailing ``nover`` set to 1, assigned in that
order (one window: only the trailing ones; ``nover = 0``: ``tap[-0:]``, the whole taper, which is ones then).
Traces past the last window are 0 in the forward and ignored in the adjoint."""
import numpy as np

from .. import LinearOperator
from ..utils.tapers import taper2d


def _slidingsteps(ntr, nwin, nover):
    if nwin > ntr:
        raise ValueError(f"nwin={nwin} is bigger than ntr={ntr}...")
    if nover >= nwin:
        raise ValueError(f"nover={nover} must be smaller than nwin={nwin}")
    step = nwin - nover
    starts = np.arange(0, ntr - nwin + 1, step, dtype=int)
    return starts, starts + nwin


def sliding2d_design(dimsd, nwin, nover, nop):
    """(nwins, dims, mwins_inends, dwins_inends) of a Sliding2D on data ``dimsd`` with inner model ``nop``"""
    dwin_ins, dwin_ends = _slidingsteps(dimsd[0], nwin, nover)
    nwins = len(dwin_ins)
    dims = (nwins * nop[0], nop[1])
    mwin_ins, mwin_ends = _slidingsteps(dims[0], nop[0], 0)
    return nwins, dims, ((mwin_ins, mwin_ends), (0, dims[-1])), ((dwin_ins, dwin_ends), (0, dimsd[-1]))


def window_tapers(nwins, nt, nwin, nover, tapertype):
    """the per-window tapers, pylops' dict of ``taper2d`` copies (None: no taper)"""
    if tapertype is None:
        return None
    tap = taper2d(nt, nwin, nover, tapertype=tapertype)
    tapin, tapend = tap.copy(), tap.copy()
    tapin[:nover] = 1
    tapend[-nover:] = 1
    taps = {0: tapin}
    for i in range(1, nwins - 1):
        taps[i] = tap
    taps[nwins - 1] = tapend
    return [taps[i] for i in range(nwins)]


class _Sliding(LinearOperator):
    """the shared apply: window grid starts (s0, s1) with per-window tapers of the window's data shape, the inner
    HStack summing along axis 1 and the outer along axis 0 (2-D: one window along a singleton axis)"""

    def _finish(self, Op, dimsd, wshape, starts, taps, name):
        self.Op, self.dimsd, self.wshape, self.starts, self.taps, self.name = Op, tuple(dimsd), wshape, starts, taps, name
        super().__init__(dtype=np.dtype(Op.dtype), shape=(int(np.prod(self.dimsd)), int(np.prod(self.dims))))

    def _tap(self, w):
        return None if self.taps is None else self.taps[w].astype(self.Op.dtype)

    def _matvec(self, x):
        x = np.asarray(x)
        nm = self.Op.shape[1]
        s0, s1 = self.starts
        out = None
        for i0, a in enumerate(s0):
            row = None
            for i1, b in enumerate(s1):
                w = i0 * len(s1) + i1
                v = np.asarray(self.Op.matvec(x[w * nm:(w + 1) * nm])).reshape(self.wshape)
                tap = self._tap(w)
                if tap is not None:
                    v = tap * v
                if out is None:
                    out = np.zeros(self.dimsd3, dtype=v.dtype)
                if row is None:
                    row = np.zeros((self.wshape[0],) + self.dimsd3[1:], dtype=v.dtype)
                row[:, b:b + self.wshape[1]] += v
            out[a:a + self.wshape[0]] += row
        return out.ravel()

    def _rmatvec(self, y):
        y = np.asarray(y).reshape(self.dimsd3)
        s0, s1 = self.starts
        parts = []
        for i0, a in enumerate(s0):
            for i1, b in enumerate(s1):
                w = i0 * len(s1) + i1
                d = y[a:a + self.wshape[0], b:b + self.wshape[1]]
                tap = self._tap(w)
                if tap is not None:
                    d = tap * d
                parts.append(np.asarray(self.Op.rmatvec(d.ravel())))
        return np.concatenate(parts)


class Sliding2D(_Sliding):
    """Sliding2D(Op, dims, dimsd, nwin, nover, tapertype="hanning", name="S")"""

    def __init__(self, Op, dims, dimsd, nwin, nover, tapertype="hanning", name="S"):
        dims, dimsd = tuple(int(d) for d in dims), tuple(int(d) for d in dimsd)
        starts, _ = _slidingsteps(dimsd[0], nwin, nover)
        nwins = len(starts)
        if nwins * Op.shape[1] // dims[1] != dims[0]:
            raise ValueError(f"Model shape (dims={dims}) is not consistent with chosen number of windows. Run "
                             f"sliding2d_design to identify the correct number of windows for the current model size...")
        if Op.shape[0] != nwin * dimsd[1]:
            raise ValueError(f"Op has {Op.shape[0]} data values, a window {nwin} x {dimsd[1]}")
        self.dims, self.nwin, self.nover, self.tapertype = dims, nwin, nover, tapertype
        self.dimsd3 = (1,) + dimsd
        taps = window_tapers(nwins, dimsd[1], nwin, nover, tapertype)
        self._finish(Op, dimsd, (1, nwin, dimsd[1]), (np.zeros(1, dtype=int), starts),
                     None if taps is None else [t[np.newaxis] for t in taps], name)
