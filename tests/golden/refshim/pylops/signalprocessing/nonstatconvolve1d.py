"""Restatement of third-party ``pylops.signalprocessing.NonStationaryConvolve1D`` -- TEST INFRASTRUCTURE for
tests/golden/make_golden_nsconvolve.py (imported as ``pylops.signalprocessing.nonstatconvolve1d``)."""
import numpy as np

from .._algebra import AlgebraOperator


class NonStationaryConvolve1D(AlgebraOperator):
    """Restatement of third-party ``pylops.signalprocessing.NonStationaryConvolve1D`` (pylops 2.x, as remembered:
    pylops is not installed here) -- TEST INFRASTRUCTURE so that the reference's MPIBlockDiag and ISTA can be run
    over a rank-local non-stationary convolution.  ``hs`` (nfilt, nh) holds filters of odd length at the regularly
    spaced samples ``ih``; pylops' loop over the model samples ``ix`` along ``axis`` interpolates ``h_ix``
    (:meth:`_interpolate_h`) and spreads ``h_ix * x[ix]`` onto ``y[ix - nh // 2 : ix + nh // 2 + 1]`` (forward), or
    gathers ``y[ix] = sum(h_ix * x[window])`` (adjoint)."""

    def __init__(self, dims, hs, ih, axis=-1, dtype="float64"):
        hs = np.asarray(hs)
        ih = np.asarray(ih)
        self.dims = tuple(int(d) for d in (dims if np.ndim(dims) else (dims,)))
        self.axis = axis % len(self.dims)
        if hs.shape[1] % 2 == 0:
            raise ValueError("filters hs must have odd length")
        if len(ih) != hs.shape[0]:
            raise ValueError("ih must hold one index per filter")
        if len(np.unique(np.diff(ih))) > 1:
            raise ValueError("the indices of filters 'ih' are must be regularly sampled")
        if min(ih) < 0 or max(ih) >= self.dims[self.axis]:
            raise ValueError("the indices of filters 'ih' must be larger than 0 and smaller than `dims`")
        self.hs = hs
        self.hsize = hs.shape[1]
        self.oh, self.dh, self.nh = int(ih[0]), int(ih[1] - ih[0]) if len(ih) > 1 else 1, len(ih)
        n = int(np.prod(self.dims))
        super().__init__(dtype=np.dtype(dtype), shape=(n, n))

    @staticmethod
    def _interpolate_h(hs, ix, oh, dh, nh):
        """filter of sample ``ix``: pylops' scalar arithmetic (a Python float weight times a row of ``hs``)"""
        ih_closest = int(np.floor((ix - oh) / dh))
        if ih_closest < 0:
            h = hs[0]
        elif ih_closest + 1 >= nh:
            h = hs[nh - 1]
        else:
            dh_closest = (ix - oh) / dh - ih_closest
            h = (1 - dh_closest) * hs[ih_closest] + dh_closest * hs[ih_closest + 1]
        return h

    def _matvec_rmatvec(self, x, rmatvec):
        x = np.moveaxis(np.reshape(x, self.dims), self.axis, 0)
        y = np.zeros(x.shape, dtype=np.result_type(x.dtype, self.dtype))
        n, hc = x.shape[0], self.hsize // 2
        for ix in range(n):
            h = self._interpolate_h(self.hs, ix, self.oh, self.dh, self.nh)
            xlo, xhi = max(0, ix - hc), min(ix + hc + 1, n)
            hlo, hhi = max(0, hc - ix), min(self.hsize, hc + (n - ix))
            hw = h[hlo:hhi].reshape((-1,) + (1,) * (x.ndim - 1))
            if not rmatvec:
                y[xlo:xhi] += hw * x[ix]
            else:
                y[ix] = np.sum(hw * x[xlo:xhi], axis=0)
        return np.moveaxis(y, 0, self.axis).ravel()

    def _matvec(self, x):
        return self._matvec_rmatvec(x, False)

    def _rmatvec(self, x):
        return self._matvec_rmatvec(x, True)
