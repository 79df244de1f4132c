"""Restatement of third-party ``pylops.signalprocessing.NonStationaryConvolve3D`` -- TEST INFRASTRUCTURE for
tests/golden/make_golden_nsconvolve3d.py (imported as ``pylops.signalprocessing.nonstatconvolve3d``)."""
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


class NonStationaryConvolve3D(AlgebraOperator):
    """Restatement of third-party ``pylops.signalprocessing.NonStationaryConvolve3D`` (pylops 2.x, engine="numpy", as
    remembered: pylops is not installed here) -- TEST INFRASTRUCTURE so that the reference's MPIBlockDiag and cgls
    can be run over a rank-local non-stationary 3-D convolution.  ``hs`` (nfx, nfy, nfz, nhx, nhy, nhz) holds filters
    of odd sizes at the regularly spaced points ``(ihx[a], ihy[b], ihz[e])``; pylops' loop over the model points
    ``(ix, iy, iz)`` interpolates ``h`` trilinearly (:meth:`weights`, :meth:`interpolate_h`: eight terms, each
    weight the float64 product ``wz * wy * wx`` taken left to right) and spreads ``h * x[ix, iy, iz]`` onto the volume
    window around the point, cut at the edges (forward), or gathers ``y[ix, iy, iz] = sum(h * x[window])``
    (adjoint)."""

    def __init__(self, dims, hs, ihx, ihy, ihz, engine="numpy", num_threads_per_blocks=(2, 16, 16),
                 dtype="float64"):
        hs = np.asarray(hs)
        self.dims = tuple(int(d) for d in dims)
        if hs.shape[3] % 2 == 0 or hs.shape[4] % 2 == 0 or hs.shape[5] % 2 == 0:
            raise ValueError("filters hs must have odd length")
        self.ohx, self.dhx = _regular("ihx", np.asarray(ihx), hs.shape[0], self.dims[0])
        self.ohy, self.dhy = _regular("ihy", np.asarray(ihy), hs.shape[1], self.dims[1])
        self.ohz, self.dhz = _regular("ihz", np.asarray(ihz), hs.shape[2], self.dims[2])
        self.hs = hs
        self.hshape = hs.shape[3:]
        n = self.dims[0] * self.dims[1] * self.dims[2]
        super().__init__(dtype=np.dtype(dtype), shape=(n, n))

    @staticmethod
    def weights(i, oh, dh, nf):
        """pylops' per-axis interpolation of point ``i``: (left filter, right filter, their weights); outside the
        nodes both are the end filter, with weights 0.5 and 0.5"""
        il = int(np.floor((i - oh) / dh))
        dr = (i - oh) / dh - il
        if il < 0:
            return 0, 0, 0.5, 0.5
        if il >= nf - 1:
            return nf - 1, nf - 1, 0.5, 0.5
        return il, il + 1, 1.0 - dr, dr

    def interpolate_h(self, ix, iy, iz):
        hs = self.hs
        ihx_l, ihx_r, dhx_l, dhx_r = self.weights(ix, self.ohx, self.dhx, hs.shape[0])
        ihy_l, ihy_r, dhy_l, dhy_r = self.weights(iy, self.ohy, self.dhy, hs.shape[1])
        ihz_l, ihz_r, dhz_l, dhz_r = self.weights(iz, self.ohz, self.dhz, hs.shape[2])
        return (dhz_l * dhy_l * dhx_l * hs[ihx_l, ihy_l, ihz_l] + dhz_r * dhy_l * dhx_l * hs[ihx_l, ihy_l, ihz_r]
                + dhz_l * dhy_r * dhx_l * hs[ihx_l, ihy_r, ihz_l] + dhz_r * dhy_r * dhx_l * hs[ihx_l, ihy_r, ihz_r]
                + dhz_l * dhy_l * dhx_r * hs[ihx_r, ihy_l, ihz_l] + dhz_r * dhy_l * dhx_r * hs[ihx_r, ihy_l, ihz_r]
                + dhz_l * dhy_r * dhx_r * hs[ihx_r, ihy_r, ihz_l] + dhz_r * dhy_r * dhx_r * hs[ihx_r, ihy_r, ihz_r])

    def _matvec_rmatvec(self, x, rmatvec):
        x = np.reshape(x, self.dims)
        y = np.zeros(self.dims, dtype=np.result_type(x.dtype, self.dtype))
        (nx, ny, nz), (nhx, nhy, nhz) = self.dims, self.hshape
        hcx, hcy, hcz = nhx // 2, nhy // 2, nhz // 2
        for ix in range(nx):
            x0, x1 = max(0, ix - hcx), min(ix + hcx + 1, nx)
            hx0, hx1 = max(0, hcx - ix), min(nhx, hcx + (nx - ix))
            for iy in range(ny):
                y0, y1 = max(0, iy - hcy), min(iy + hcy + 1, ny)
                hy0, hy1 = max(0, hcy - iy), min(nhy, hcy + (ny - iy))
                for iz in range(nz):
                    h = self.interpolate_h(ix, iy, iz)
                    z0, z1 = max(0, iz - hcz), min(iz + hcz + 1, nz)
                    hz0, hz1 = max(0, hcz - iz), min(nhz, hcz + (nz - iz))
                    if rmatvec:
                        y[ix, iy, iz] = np.sum(h[hx0:hx1, hy0:hy1, hz0:hz1] * x[x0:x1, y0:y1, z0:z1])
                    else:
                        y[x0:x1, y0:y1, z0:z1] += h[hx0:hx1, hy0:hy1, hz0:hz1] * x[ix, iy, iz]
        return y.ravel()

    def _matvec(self, x):
        return self._matvec_rmatvec(x, False)

    def _rmatvec(self, x):
        return self._matvec_rmatvec(x, True)
