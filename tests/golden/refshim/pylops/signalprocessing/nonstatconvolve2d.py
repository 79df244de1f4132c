"""Restatement of third-party ``pylops.signalprocessing.NonStationaryConvolve2D`` -- TEST INFRASTRUCTURE for
tests/golden/make_golden_nsconvolve2d.py (imported as ``pylops.signalprocessing.nonstatconvolve2d``)."""
import numpy as np

from .._algebra import AlgebraOperator


def _regular(name, ih, nf, n):
    if len(ih) != nf:
        raise ValueError(f"{name} must hold one index per filter")
    if len(np.unique(np.diff(ih))) > 1:
        raise ValueError(f"the indices of filters '{name}' are must be regularly sampled")
    if min(ih) < 0 or max(ih) >= n:
        raise ValueError(f"the indices of filters '{name}' must be larger than 0 and smaller than `dims`")
    return int(ih[0]), int(ih[1] - ih[0]) if len(ih) > 1 else 1


class NonStationaryConvolve2D(AlgebraOperator):
    """Restatement of third-party ``pylops.signalprocessing.NonStationaryConvolve2D`` (pylops 2.x, engine="numpy", as
    remembered: pylops is not installed here) -- TEST INFRASTRUCTURE so that the reference's MPIBlockDiag and cgls
    can be run over a rank-local non-stationary 2-D convolution.  ``hs`` (nfx, nfz, nhx, nhz) holds filters of odd
    sizes at the regularly spaced points ``(ihx[a], ihz[b])``; pylops' loop over the model points ``(ix, iz)``
    interpolates ``h`` bilinearly (:meth:`weights`, :meth:`interpolate_h`) and spreads ``h * x[ix, iz]`` onto the
    image window around the point, cut at the edges (forward), or gathers ``y[ix, iz] = sum(h * x[window])``
    (adjoint)."""

    def __init__(self, dims, hs, ihx, ihz, engine="numpy", num_threads_per_blocks=(32, 32), dtype="float64"):
        hs = np.asarray(hs)
        self.dims = tuple(int(d) for d in dims)
        if hs.shape[2] % 2 == 0 or hs.shape[3] % 2 == 0:
            raise ValueError("filters hs must have odd length")
        self.ohx, self.dhx = _regular("ihx", np.asarray(ihx), hs.shape[0], self.dims[0])
        self.ohz, self.dhz = _regular("ihz", np.asarray(ihz), hs.shape[1], self.dims[1])
        self.hs = hs
        self.hshape = hs.shape[2:]
        n = self.dims[0] * self.dims[1]
        super().__init__(dtype=np.dtype(dtype), shape=(n, n))

    @staticmethod
    def weights(i, oh, dh, nf):
        """pylops' per-axis interpolation of point ``i``: (left / top filter, right / bottom filter, their weights);
        outside the nodes both are the end filter, with weights 0.5 and 0.5"""
        il = int(np.floor((i - oh) / dh))
        dr = (i - oh) / dh - il
        if il < 0:
            return 0, 0, 0.5, 0.5
        if il >= nf - 1:
            return nf - 1, nf - 1, 0.5, 0.5
        return il, il + 1, 1.0 - dr, dr

    def interpolate_h(self, ix, iz):
        hs = self.hs
        ihx_l, ihx_r, dhx_l, dhx_r = self.weights(ix, self.ohx, self.dhx, hs.shape[0])
        ihz_t, ihz_b, dhz_t, dhz_b = self.weights(iz, self.ohz, self.dhz, hs.shape[1])
        h_tl, h_bl = hs[ihx_l, ihz_t], hs[ihx_l, ihz_b]
        h_tr, h_br = hs[ihx_r, ihz_t], hs[ihx_r, ihz_b]
        return dhz_t * dhx_l * h_tl + dhz_b * dhx_l * h_bl + dhz_t * dhx_r * h_tr + dhz_b * dhx_r * h_br

    def _matvec_rmatvec(self, x, rmatvec):
        x = np.reshape(x, self.dims)
        y = np.zeros(self.dims, dtype=np.result_type(x.dtype, self.dtype))
        (nx, nz), (nhx, nhz) = self.dims, self.hshape
        hcx, hcz = nhx // 2, nhz // 2
        for ix in range(nx):
            for iz in range(nz):
                h = self.interpolate_h(ix, iz)
                x0, x1 = max(0, ix - hcx), min(ix + hcx + 1, nx)
                z0, z1 = max(0, iz - hcz), min(iz + hcz + 1, nz)
                hx0, hx1 = max(0, hcx - ix), min(nhx, hcx + (nx - ix))
                hz0, hz1 = max(0, hcz - iz), min(nhz, hcz + (nz - iz))
                if rmatvec:
                    y[ix, iz] = np.sum(h[hx0:hx1, hz0:hz1] * x[x0:x1, z0:z1])
                else:
                    y[x0:x1, z0:z1] += h[hx0:hx1, hz0:hz1] * x[ix, iz]
        return y.ravel()

    def _matvec(self, x):
        return self._matvec_rmatvec(x, False)

    def _rmatvec(self, x):
        return self._matvec_rmatvec(x, True)
