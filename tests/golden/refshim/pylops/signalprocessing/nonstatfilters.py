"""Restatement of third-party ``pylops.signalprocessing.NonStationaryFilters1D`` / ``NonStationaryFilters2D`` -- TEST
INFRASTRUCTURE for tests/golden/make_golden_nsfilters.py (imported as ``pylops.signalprocessing.nonstatfilters``)."""
import numpy as np

from .._algebra import AlgebraOperator
from .nonstatconvolve1d import NonStationaryConvolve1D
from .nonstatconvolve2d import NonStationaryConvolve2D, _regular


class NonStationaryFilters1D(AlgebraOperator):
    """Restatement of third-party ``pylops.signalprocessing.NonStationaryFilters1D`` (pylops 2.x, as remembered:
    pylops is not installed here) -- TEST INFRASTRUCTURE so that the reference's MPIVStack and cgls can be run over a
    rank-local non-stationary filter estimation.  The model is the bank ``(len(ih), hsize)``; pylops' loop over the
    samples ``ix`` of the fixed 1-D ``inp`` interpolates ``h_ix`` from the model (``NonStationaryConvolve1D.
    _interpolate_h``) and spreads ``inp[ix] * h_ix`` onto the window around ``ix`` (forward), or adds
    ``w * inp[ix] * y[window]`` to each filter around ``ix`` with its interpolation weight ``w`` (adjoint)."""

    def __init__(self, inp, hsize, ih, dtype="float64", name="C"):
        self.inp, ih = np.asarray(inp), np.asarray(ih)
        if hsize % 2 == 0:
            raise ValueError("filters hs must have odd length")
        n = self.inp.size
        self.oh, self.dh = _regular("ih", ih, len(ih), n)
        self.nh, self.hsize = len(ih), int(hsize)
        self.dims, self.dimsd = (self.nh, self.hsize), (n,)
        super().__init__(dtype=np.dtype(dtype), shape=(n, self.nh * self.hsize))

    def _window(self, ix):
        n, hc = self.inp.size, self.hsize // 2
        return slice(max(0, ix - hc), min(ix + hc + 1, n)), slice(max(0, hc - ix), min(self.hsize, hc + (n - ix)))

    def _matvec(self, x):
        hs = np.reshape(x, self.dims)
        y = np.zeros(self.inp.size, dtype=np.result_type(hs.dtype, self.inp.dtype, self.dtype))
        for ix in range(self.inp.size):
            h = NonStationaryConvolve1D._interpolate_h(hs, ix, self.oh, self.dh, self.nh)
            win, cut = self._window(ix)
            y[win] += self.inp[ix] * h[cut]
        return y

    def _rmatvec(self, x):
        hs = np.zeros(self.dims, dtype=np.result_type(x.dtype, self.inp.dtype, self.dtype))
        for ix in range(self.inp.size):
            win, cut = self._window(ix)
            htmp = self.inp[ix] * x[win]
            il = int(np.floor((ix - self.oh) / self.dh))
            if il < 0:
                hs[0, cut] += htmp
            elif il + 1 >= self.nh:
                hs[self.nh - 1, cut] += htmp
            else:
                dr = (ix - self.oh) / self.dh - il
                hs[il, cut] += (1 - dr) * htmp
                hs[il + 1, cut] += dr * htmp
        return hs.ravel()


class NonStationaryFilters2D(AlgebraOperator):
    """Restatement of third-party ``pylops.signalprocessing.NonStationaryFilters2D`` (pylops 2.x, engine="numpy", as
    remembered: pylops is not installed here) -- TEST INFRASTRUCTURE so that the reference's MPIVStack and cgls can be
    run over a rank-local non-stationary filter estimation.  The model is the bank ``(nfx, nfz, nhx, nhz)``; pylops'
    loop over the points ``(ix, iz)`` of the fixed image ``inp`` interpolates ``h`` bilinearly from the model
    (``NonStationaryConvolve2D.weights``) and spreads ``inp[ix, iz] * h`` onto the image window around the point, cut
    at the edges (forward), or adds ``w * inp[ix, iz] * y[window]`` to each of the four filters around the point with
    its weight ``w = wz * wx`` (adjoint; outside the nodes the four are the end filter, at a quarter each)."""

    def __init__(self, inp, hshape, ihx, ihz, engine="numpy", num_threads_per_blocks=(32, 32), dtype="float64",
                 name="C"):
        self.inp = np.asarray(inp)
        self.hshape = tuple(int(h) for h in hshape)
        if self.hshape[0] % 2 == 0 or self.hshape[1] % 2 == 0:
            raise ValueError("filters hs must have odd length")
        nx, nz = self.inp.shape
        self.ohx, self.dhx = _regular("ihx", np.asarray(ihx), len(ihx), nx)
        self.ohz, self.dhz = _regular("ihz", np.asarray(ihz), len(ihz), nz)
        self.nf = (len(ihx), len(ihz))
        self.dims, self.dimsd = self.nf + self.hshape, (nx, nz)
        super().__init__(dtype=np.dtype(dtype), shape=(nx * nz, int(np.prod(self.dims))))

    def _windows(self, ix, iz):
        (nx, nz), (nhx, nhz) = self.dimsd, self.hshape
        hcx, hcz = nhx // 2, nhz // 2
        win = (slice(max(0, ix - hcx), min(ix + hcx + 1, nx)), slice(max(0, iz - hcz), min(iz + hcz + 1, nz)))
        cut = (slice(max(0, hcx - ix), min(nhx, hcx + (nx - ix))), slice(max(0, hcz - iz), min(nhz, hcz + (nz - iz))))
        return win, cut

    def _four(self, ix, iz):
        """[(a, b, weight)] of the four filters around (ix, iz), in pylops' order"""
        xl, xr, wxl, wxr = NonStationaryConvolve2D.weights(ix, self.ohx, self.dhx, self.nf[0])
        zt, zb, wzt, wzb = NonStationaryConvolve2D.weights(iz, self.ohz, self.dhz, self.nf[1])
        return [(xl, zt, wzt * wxl), (xl, zb, wzb * wxl), (xr, zt, wzt * wxr), (xr, zb, wzb * wxr)]

    def _matvec(self, x):
        hs = np.reshape(x, self.dims)
        y = np.zeros(self.dimsd, dtype=np.result_type(hs.dtype, self.inp.dtype, self.dtype))
        for ix in range(self.dimsd[0]):
            for iz in range(self.dimsd[1]):
                h = sum(w * hs[a, b] for a, b, w in self._four(ix, iz))
                win, cut = self._windows(ix, iz)
                y[win] += self.inp[ix, iz] * h[cut]
        return y.ravel()

    def _rmatvec(self, x):
        x = np.reshape(x, self.dimsd)
        hs = np.zeros(self.dims, dtype=np.result_type(x.dtype, self.inp.dtype, self.dtype))
        for ix in range(self.dimsd[0]):
            for iz in range(self.dimsd[1]):
                win, cut = self._windows(ix, iz)
                htmp = self.inp[ix, iz] * x[win]
                for a, b, w in self._four(ix, iz):
                    hs[a, b][cut] += w * htmp
        return hs.ravel()
