"""Restatement of third-party ``pylops.signalprocessing.Patch2D`` (pylops 2.x, as remembered: pylops is not installed
here to check it) -- TEST INFRASTRUCTURE so that the reference's MPIBlockDiag and FISTA can be run over time-space
patch operators by tests/golden/make_golden_patch.py.  ``_Patches`` is the chain shared with Sliding1D (sliding1d.py)
and Patch3D (patch3d.py).

Patches ``nwin = (nwin0, nwin1)`` overlapping by ``nover`` run along both axes of the data ``dimsd = (n, nt)``,
starting every ``nwin - nover`` (sliding2d's ``_slidingsteps`` per axis); patch ``w = i0 * nwins1 + i1``.  The model is
``(nwins0 * nop[0], nwins1 * nop[1])`` stored window-major, as BlockDiag orders its blocks.  pylops builds
``HStack_0 * BlockDiag([HStack_1] * nwins0) * BlockDiag([Diagonal(tap_w) * Op])``, HStack_1 placing the patches of
row i0 along t in a strip of nwin0 traces and HStack_0 placing the strips along the traces; this restatement applies
that chain in its order, one HStack level per window axis:

    strip_i0 = 0;  for i1 ascending:  strip_i0[:, t_i1] += tap_w * Op.matvec(x_w)        (tap_w of Op's dtype)
    y = 0;         for i0 ascending:  y[h_i0] += strip_i0
    x_w = Op.rmatvec(tap_w * d[h_i0, t_i1])

Remembered items: ``patch2d_design`` and its return; the ``ValueError`` of a model ``dims`` other than
``(nwins0 * nop[0], nwins1 * nop[1])`` (and, restated here, of an ``Op`` whose model is not ``nop`` or whose data are
not a patch); the tapers ``taper2d(nwin[1], nwin[0], nover, tapertype)`` (a pair ``nover``), the outer product of
the two axis tapers, with the edge patches' outer ``nover`` rows (axis 0) / columns (axis 1) replaced by the taper's
middle row ``nwin[0] // 2`` / column ``nwin[1] // 2``, assigned in pylops' order -- top, bottom, left, right, then
the four corners -- so that one patch along an axis keeps only its trailing edge replaced and ``nover = 0`` hits
``[-0:]`` (the whole middle row / column); ``scalings`` (None only here) and ``savetaper`` are not restated.  Traces and
samples past the last patch are 0 in the forward and ignored in the adjoint."""
import numpy as np

from .. import LinearOperator
from ..utils.tapers import taper
from .sliding2d import _slidingsteps


def _design(dimsd, nwin, nover, nop):
    d = [_slidingsteps(dimsd[a], nwin[a], nover[a]) for a in range(len(nwin))]
    nwins = tuple(len(di[0]) for di in d)
    dims = tuple(nw * n for nw, n in zip(nwins, nop))
    m = [_slidingsteps(dims[a], nop[a], 0) for a in range(len(nwin))]
    return nwins, dims, tuple(m), tuple(d)


def patch2d_design(dimsd, nwin, nover, nop):
    """(nwins, dims, mwins_inends, dwins_inends) of a Patch2D on data ``dimsd`` with inner model ``nop``"""
    return _design(dimsd, nwin, nover, nop)


def edge_tapers(tap, nwins0, nwins1, nwin, nover):
    """pylops' per-patch tapers of a patch grid: ``tap`` (axes 0 and 1 the grid's) with the edge rows / columns
    replaced by the middle row / column, in pylops' order"""
    nwins = nwins0 * nwins1
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
            t[:, :nover[1]] = t[:, mid1:mid1 + 1]
        else:
            t[:, -nover[1]:] = t[:, mid1:mid1 + 1]
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


def taper2d(nt, nmask, ntap, tapertype="hanning"):
    """pylops.utils.tapers.taper2d with a pair ``ntap``, as Patch2D calls it: the outer product of the taper of
    ``nmask`` samples over ``ntap[0]`` and the taper of ``nt`` samples over ``ntap[1]`` (utils/tapers.py restates the
    integer form, a taper tiled along the second axis)"""
    return np.outer(taper(nmask, ntap[0], tapertype), taper(nt, ntap[1], tapertype))


def window_tapers(nwins0, nwins1, nwin, nover, tapertype):
    """the per-patch tapers (None: no taper)"""
    if tapertype is None:
        return None
    return edge_tapers(taper2d(nwin[1], nwin[0], tuple(nover), tapertype=tapertype), nwins0, nwins1, nwin, nover)


class _Patches(LinearOperator):
    """the chain of nested HStacks over windows ``wshape`` on every axis of ``dimsd``, window starts ``starts[k]``
    along axis k, window w the row-major index of its per-axis indices, per-window tapers ``taps`` (None: none)"""

    def _finish(self, Op, dims, dimsd, wshape, starts, taps, name):
        self.Op, self.dims, self.dimsd, self.wshape = Op, tuple(dims), tuple(dimsd), tuple(wshape)
        self.starts, self.taps, self.name = starts, taps, name
        self.nwins = tuple(len(s) for s in starts)
        super().__init__(dtype=np.dtype(Op.dtype), shape=(int(np.prod(self.dimsd)), int(np.prod(self.dims))))

    def _tap(self, w):
        return None if self.taps is None else self.taps[w].astype(self.Op.dtype)

    def _window(self, idx):
        return int(np.ravel_multi_index(idx, self.nwins))

    def _matvec(self, x):
        x = np.asarray(x)
        nm, K = self.Op.shape[1], len(self.wshape)

        def level(k, idx):
            """HStack k: the windows idx + (i,) placed along axis k of a strip wshape[:k] + dimsd[k:]"""
            out = None
            for i, a in enumerate(self.starts[k]):
                if k == K - 1:
                    w = self._window(idx + (i,))
                    v = np.asarray(self.Op.matvec(x[w * nm:(w + 1) * nm])).reshape(self.wshape)
                    tap = self._tap(w)
                    if tap is not None:
                        v = tap * v
                else:
                    v = level(k + 1, idx + (i,))
                if out is None:
                    out = np.zeros(self.wshape[:k] + self.dimsd[k:], dtype=v.dtype)
                out[(slice(None),) * k + (slice(a, a + self.wshape[k]),)] += v
            return out
        return level(0, ()).ravel()

    def _rmatvec(self, y):
        y = np.asarray(y).reshape(self.dimsd)
        parts = []
        for idx in np.ndindex(*self.nwins):
            w = self._window(idx)
            d = y[tuple(slice(s[i], s[i] + n) for s, i, n in zip(self.starts, idx, self.wshape))]
            tap = self._tap(w)
            if tap is not None:
                d = tap * d
            parts.append(np.asarray(self.Op.rmatvec(d.ravel())))
        return np.concatenate(parts)


def check(Op, dims, nwins, nop, wshape, design):
    if tuple(dims) != tuple(nw * n for nw, n in zip(nwins, nop)):
        raise ValueError(f"Model shape (dims={dims}) is not consistent with chosen number of windows. Run "
                         f"{design} to identify the correct number of windows for the current model size...")
    if Op.shape[1] != int(np.prod(nop)):
        raise ValueError(f"Op has {Op.shape[1]} model values, nop {nop}")
    if Op.shape[0] != int(np.prod(wshape)):
        raise ValueError(f"Op has {Op.shape[0]} data values, a window {wshape}")


class Patch2D(_Patches):
    """Patch2D(Op, dims, dimsd, nwin, nover, nop, tapertype="hanning", scalings=None, name="P")"""

    def __init__(self, Op, dims, dimsd, nwin, nover, nop, tapertype="hanning", scalings=None, name="P"):
        dims, dimsd = tuple(int(d) for d in dims), tuple(int(d) for d in dimsd)
        nwin, nover, nop = tuple(int(v) for v in nwin), tuple(int(v) for v in nover), tuple(int(v) for v in nop)
        if scalings is not None:
            raise NotImplementedError("scalings are not restated")
        s = [_slidingsteps(dimsd[a], nwin[a], nover[a])[0] for a in (0, 1)]
        check(Op, dims, (len(s[0]), len(s[1])), nop, nwin, "patch2d_design")
        self.nwin, self.nover, self.nop, self.tapertype = nwin, nover, nop, tapertype
        self._finish(Op, dims, dimsd, nwin, s, window_tapers(len(s[0]), len(s[1]), nwin, nover, tapertype), name)
