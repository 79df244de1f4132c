"""Restatement of third-party ``pylops.signalprocessing.Convolve1D`` -- TEST INFRASTRUCTURE for
tests/golden/make_golden_convolve.py (imported as ``pylops.signalprocessing.convolve1d``)."""
import numpy as np

from .. import LinearOperator


class Convolve1D(LinearOperator):
    """Restatement of third-party ``pylops.signalprocessing.Convolve1D`` (pylops 2.x, stationary 1-D filter,
    direct method) -- TEST INFRASTRUCTURE so that the reference's MPIBlockDiag and ISTA can be run over the
    rank-local convolution of tutorials/reflectivity.py by tests/golden/make_golden_convolve.py.  As pylops
    computes it: ``h`` is padded by ``2 * (nh // 2 - offset)`` zeros (one fewer when ``nh`` is even) in front, or
    behind when that count is negative, then ``scipy.signal.convolve(..., mode="same")`` is applied along ``axis``
    forward and ``scipy.signal.correlate(..., mode="same")`` for the adjoint."""

    def __init__(self, dims, h, offset=0, axis=-1, method=None, dtype="float64"):
        h = np.asarray(h)
        if h.ndim != 1:
            raise NotImplementedError("non-stationary filters are not restated")
        self.dims = tuple(int(d) for d in (dims if np.ndim(dims) else (dims,)))
        self.axis = axis % len(self.dims)
        self.nh = h.size
        if not 0 <= offset <= self.nh - 1:
            raise ValueError("offset must be in [0, nh - 1]")
        pad = 2 * (self.nh // 2 - int(offset))
        if self.nh % 2 == 0:
            pad -= 1
        if pad != 0:
            h = np.pad(h, (pad if pad > 0 else 0, -pad if pad < 0 else 0), mode="constant")
        self.h = h
        n = int(np.prod(self.dims))
        super().__init__(dtype=np.dtype(dtype), shape=(n, n))

    def _along(self, x, fn):
        import scipy.signal
        x = np.reshape(x, self.dims)
        y = np.apply_along_axis(lambda v: fn(v, self.h, mode="same", method="direct"), self.axis, x)
        return y.ravel()

    def _matvec(self, x):
        import scipy.signal
        return self._along(x, scipy.signal.convolve)

    def _rmatvec(self, x):
        import scipy.signal
        return self._along(x, scipy.signal.correlate)
