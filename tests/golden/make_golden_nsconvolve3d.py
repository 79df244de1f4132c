"""Generate the non-stationary 3-D convolution fixtures by running the REAL reference's MPIBlockDiag and cgls (a
pylops-mpi checkout named by PYLOPS_MPI_REFERENCE, imported unmodified through make_golden.load_reference) over
refshim's restated ``pylops.signalprocessing.NonStationaryConvolve3D`` (refshim/pylops/signalprocessing/
nonstatconvolve3d.py) and, for the point-spread functions, refshim's 3-D ``pylops.waveeqprocessing.Kirchhoff``
(refshim/pylops/waveeqprocessing/kirchhoff3d.py).

    PYLOPS_MPI_REFERENCE=<checkout> python tests/golden/make_golden_nsconvolve3d.py   # writes nsconvolve3d_golden.npz

Operator cases.  A (NV, NX, NY, NZ) stack of volumes split along axis 0 over P in {1, 2, 3} ranks: rank r holds
MPIBlockDiag([NonStationaryConvolve3D((NX, NY, NZ), hs_k, ihx, ihy, ihz) for its volumes k]), one bank per volume.
Filter sizes ``NHS`` (1 x 1 x 1 up to 13 x 3 x 15, larger than the volume along x and z; not all cubic), banks
``BANKS`` (1 x 1 x 1 up to 3 x 3 x 3, with steps 1 and 4 mixed over the axes), ih = 1 + dh * arange(nf) on every
axis: both edges of every axis are extrapolated.  Inputs are exactly representable: x has entries in {-1, 0, 1}, the
taps are drawn from {-1, -1/2, 1/2, 1} and the steps are 1 or 4, so every trilinear weight is a multiple of 1/64,
every output a multiple of 1/128, and each is the SAME in float64, float32 and complex128 and at every P (all checked
here).  Each output is stored once, losslessly, as int32 of ENC * y.

  op/nh{nhx}x{nhy}x{nhz}/nf{nfx}x{nfy}x{nfz}/dh{dhx}x{dhy}x{dhz}/{y,ya}   gathered forward of x / adjoint of v
  .../{yi,yai}   imaginary parts of the complex128 runs, for the cases of ``complex_case``

Flow: 3-D image-domain least-squares migration.  A refshim 3-D Kirchhoff ``K`` (analytic, a (FLOW_NY, FLOW_NX,
FLOW_NZ) image) gives the point-spread functions of a grid of point scatterers at (FLOW_IHY, FLOW_IHX, FLOW_IHZ):
hs[a, b, e] = the FLOW_NH window of K^H K m_psf around node (FLOW_IHY[a], FLOW_IHX[b], FLOW_IHZ[e]), and the migrated
volumes m_mig = K^H K m_true of FLOW_NV layered reflectivities.  Then cgls(MPIBlockDiag([NSC3D(hs)] * nv_r), m_mig,
x0 = 0) for FLOW_NITER iterations (tol = 0).  ``flow/cond`` is the 2-norm condition number of the PSF operator (its
dense float64 matrix).  ``flow/spread`` is how far rounding alone moves the run: the largest change of x (relative to
max |x|) and of the cost history (relative) when every apply of the restated operator is jittered by 4 ulps, over
the seeds FLOW_JITTER_SEEDS at P = 1.  The tests derive their tolerance from both.  On this PSF bank that spread
grows about a hundredfold per iteration past the thirteenth (5e-3 in the cost after 20), so the run stops at 12
iterations, where it is still reproducible.

  flow/hs, flow/mmig, flow/cond, flow/spread, flow/P{P}/{x,iiter,cost}
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from fixture_codec import encode, rows_of  # noqa: E402

NV, NX, NY, NZ = 4, 10, 11, 13
NHS = ((1, 1, 1), (3, 5, 1), (1, 3, 7), (5, 3, 3), (13, 3, 15))
BANKS = (((1, 1, 1), (1, 1, 1)), ((2, 3, 2), (1, 4, 4)), ((2, 2, 3), (4, 1, 4)), ((3, 3, 3), (1, 4, 4)))
DTYPES = ("float64", "float32", "complex128")
ENC = 128        # stored value = ENC * y, exact in int32

FLOW_NV, FLOW_NY, FLOW_NX, FLOW_NZ, FLOW_D = 3, 13, 15, 11, 4.0
FLOW_NT, FLOW_DT, FLOW_VEL, FLOW_F0 = 81, 0.002, 1500.0, 30.0
FLOW_NH = (7, 7, 7)
FLOW_IHY, FLOW_IHX, FLOW_IHZ = (3, 9), (3, 7, 11), (3, 7)
FLOW_NITER = 12
FLOW_JITTER_SEEDS = (1, 2, 3)
REFSHIM = os.path.join(HERE, "refshim")


def complex_case(nh, bank):
    return nh == (5, 3, 3) and bank[0] == (2, 3, 2)


def cases():
    """(nh, (nf, dh), dtype)"""
    return [(nh, bank, dt) for nh in NHS for bank in BANKS for dt in DTYPES
            if dt != "complex128" or complex_case(nh, bank)]


def key(nh, bank):
    nf, dh = bank
    return "op/nh{}x{}x{}/nf{}x{}x{}/dh{}x{}x{}".format(*nh, *nf, *dh)


def nodes(bank):
    """(ihx, ihy, ihz) of a bank: 1 + dh * arange(nf) per axis"""
    nf, dh = bank
    return tuple(1 + d * np.arange(f) for f, d in zip(nf, dh))


def case_inputs(nh, bank, dt):
    """NV banks (the real dtype of dt), (ihx, ihy, ihz), and the global x / v in dtype dt"""
    nf, dh = bank
    rng = np.random.default_rng(700 + 97 * nh[0] + 31 * nh[1] + 13 * nh[2] + 7 * nf[0] + 3 * nf[1] + nf[2] + dh[1])
    hs = rng.choice([-1.0, -0.5, 0.5, 1.0], (NV,) + nf + nh).astype(np.real(np.ones(1, dt)).dtype)
    rng = np.random.default_rng(29)
    n = NV * NX * NY * NZ
    x, v, xi, vi = (rng.integers(-1, 2, n).astype(np.float64) for _ in range(4))
    if dt == "complex128":
        x, v = x + 1j * xi, v + 1j * vi
    return hs, nodes(bank), x.astype(dt), v.astype(dt)


def refshim_modules():
    """(refshim's 3-D kirchhoff, its wavelets, the restated NonStationaryConvolve3D class); refshim/ is on the path
    only while they are imported"""
    added = REFSHIM not in sys.path
    if added:
        sys.path.insert(0, REFSHIM)
    try:
        import pylops.signalprocessing.nonstatconvolve3d as nsc3
        import pylops.utils.wavelets as wavelets
        import pylops.waveeqprocessing.kirchhoff3d as kirchhoff3d
    finally:
        if added:
            sys.path.remove(REFSHIM)
    return kirchhoff3d, wavelets, nsc3.NonStationaryConvolve3D


def flow_geometry():
    """z, x, t, srcs, recs, vel, wav, wavc, y of the 3-D Kirchhoff operator whose K^H K the flow inverts (rows of
    srcs / recs: y, x, z)"""
    _, wavelets, _ = refshim_modules()
    y, x, z = np.arange(FLOW_NY) * FLOW_D, np.arange(FLOW_NX) * FLOW_D, np.arange(FLOW_NZ) * FLOW_D
    t = np.arange(FLOW_NT) * FLOW_DT
    RY, RX = np.meshgrid(np.linspace(0, y[-1], 5), np.linspace(0, x[-1], 5), indexing="ij")
    recs = np.vstack((RY.ravel(), RX.ravel(), np.zeros(RY.size)))
    SY, SX = np.meshgrid(np.linspace(2 * FLOW_D, y[-1] - 2 * FLOW_D, 2), np.linspace(2 * FLOW_D, x[-1] - 2 * FLOW_D, 2),
                         indexing="ij")
    srcs = np.vstack((SY.ravel(), SX.ravel(), np.zeros(SY.size)))
    wav, _, wavc = wavelets.ricker(t[:15], f0=FLOW_F0)
    return z, x, t, srcs, recs, FLOW_VEL, wav, int(wavc), y


def flow_models():
    """(m_psf, m_true): the point scatterers at the filter nodes, and FLOW_NV layered reflectivities"""
    m_psf = np.zeros((FLOW_NY, FLOW_NX, FLOW_NZ))
    for py in FLOW_IHY:
        for px in FLOW_IHX:
            for pz in FLOW_IHZ:
                m_psf[py, px, pz] = 1.0
    m_true = np.zeros((FLOW_NV, FLOW_NY, FLOW_NX, FLOW_NZ))
    for k in range(FLOW_NV):
        m_true[k, :, :, 3 + k] = -1.0
        m_true[k, :, :, 9 - k] = 0.5
        m_true[k, 3 + 2 * k:8 + 2 * k, 4:10, 6] = 0.75
    return m_psf, m_true


def psf_windows(m_psf_image):
    """hs[a, b, e] = the FLOW_NH window of K^H K m_psf around node (FLOW_IHY[a], FLOW_IHX[b], FLOW_IHZ[e])"""
    h0, h1, h2 = (n // 2 for n in FLOW_NH)
    hs = np.zeros((len(FLOW_IHY), len(FLOW_IHX), len(FLOW_IHZ)) + FLOW_NH)
    for a, py in enumerate(FLOW_IHY):
        for b, px in enumerate(FLOW_IHX):
            for e, pz in enumerate(FLOW_IHZ):
                hs[a, b, e] = m_psf_image[py - h0:py + h0 + 1, px - h1:px + h1 + 1, pz - h2:pz + h2 + 1]
    return hs


def flow_matrix(hs):
    """the PSF operator's dense float64 matrix, column j the window of the restatement's h_j"""
    _, _, NSC3 = refshim_modules()
    op = NSC3((FLOW_NY, FLOW_NX, FLOW_NZ), hs, FLOW_IHY, FLOW_IHX, FLOW_IHZ)
    dims, hc = (FLOW_NY, FLOW_NX, FLOW_NZ), tuple(n // 2 for n in FLOW_NH)
    M = np.zeros(dims + (int(np.prod(dims)),))
    for j, (jx, jy, jz) in enumerate(np.ndindex(*dims)):
        lo = [max(0, c - h) for c, h in zip((jx, jy, jz), hc)]
        hi = [min(n, c + h + 1) for c, n, h in zip((jx, jy, jz), dims, hc)]
        hl = [l - c + h for l, c, h in zip(lo, (jx, jy, jz), hc)]
        h = op.interpolate_h(jx, jy, jz)
        M[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2], j] = h[hl[0]:hl[0] + hi[0] - lo[0], hl[1]:hl[1] + hi[1] - lo[1],
                                                         hl[2]:hl[2] + hi[2] - lo[2]]
    return M.reshape(M.shape[-1], M.shape[-1])


def main():
    from make_golden import load_reference          # puts refshim/ (mpi4py, pylops) on the path
    from mpi4py import MPI
    from pylops.signalprocessing.nonstatconvolve3d import NonStationaryConvolve3D
    pkg, mods = load_reference()
    import importlib
    basic = importlib.import_module("pylops_mpi.optimization.basic")
    DA = pkg.DistributedArray
    BD = mods["BlockDiag"].MPIBlockDiag
    out = {}

    def t_op(rank, P, nh, bank, dt):
        hs, ih, x, v = case_inputs(nh, bank, dt)
        nv = rows_of(P, NV)
        k0 = sum(nv[:rank])
        ls = [(r * NX * NY * NZ,) for r in nv]
        Op = BD([NonStationaryConvolve3D((NX, NY, NZ), hs[k], *ih, dtype=dt) for k in range(k0, k0 + nv[rank])],
                dtype=dt)
        return {"y": (Op @ DA.to_dist(x, local_shapes=ls)).asarray(),
                "ya": (Op.H @ DA.to_dist(v, local_shapes=ls)).asarray()}

    for nh in NHS:
        for bank in BANKS:
            runs = {}
            for dt in DTYPES:
                if dt == "complex128" and not complex_case(nh, bank):
                    continue
                for P in (1, 2, 3):
                    res = MPI.run_world(P, t_op, P, nh, bank, dt)[0]
                    if P == 1:
                        runs[dt] = res
                    for n in ("y", "ya"):                  # one bank per volume: the result does not depend on P
                        assert np.array_equal(res[n], runs[dt][n])
            k = key(nh, bank)
            for n in ("y", "ya"):
                assert np.array_equal(runs["float32"][n], runs["float64"][n])
                out[f"{k}/{n}"] = encode(runs["float64"][n], ENC, np.int32)
                if "complex128" in runs:
                    assert np.array_equal(runs["complex128"][n].real, runs["float64"][n])
                    out[f"{k}/{n}i"] = encode(runs["complex128"][n].imag, ENC, np.int32)

    # flow: the PSF bank and the migrated volumes from the restated 3-D Kirchhoff, in float64
    kirchhoff3d, _, _ = refshim_modules()
    z, x, t, srcs, recs, vel, wav, wavc, y = flow_geometry()
    K = kirchhoff3d.Kirchhoff(z, x, t, srcs, recs, vel, wav, wavc, y=y, mode="analytic")
    m_psf, m_true = flow_models()
    hs = psf_windows(K.rmatvec(K.matvec(m_psf.ravel())).reshape(FLOW_NY, FLOW_NX, FLOW_NZ))
    mmig = np.stack([K.rmatvec(K.matvec(m.ravel())) for m in m_true]).ravel()
    out["flow/hs"], out["flow/mmig"] = hs, mmig
    out["flow/cond"] = np.asarray(np.linalg.cond(flow_matrix(hs)))

    class Jittered(NonStationaryConvolve3D):
        """the restated operator with every output scaled by 1 + 4 u g, g standard normal from a seeded generator"""

        def __init__(self, seed, *args):
            super().__init__(*args)
            self.rng = np.random.default_rng(seed)

        def _jitter(self, y):
            return y * (1 + 4 * 2.0 ** -53 * self.rng.standard_normal(y.shape))

        def _matvec(self, x):
            return self._jitter(super()._matvec(x))

        def _rmatvec(self, x):
            return self._jitter(super()._rmatvec(x))

    def t_flow(rank, P, seed=None):
        nv = rows_of(P, FLOW_NV)
        ls = [(r * FLOW_NY * FLOW_NX * FLOW_NZ,) for r in nv]
        args = ((FLOW_NY, FLOW_NX, FLOW_NZ), hs, FLOW_IHY, FLOW_IHX, FLOW_IHZ)
        op = NonStationaryConvolve3D(*args) if seed is None else Jittered(seed, *args)
        Op = BD([op] * nv[rank])
        d = DA.to_dist(mmig, local_shapes=ls)
        x0 = DA(global_shape=mmig.size, local_shapes=ls)
        x0[:] = 0
        xinv, istop, iiter, r1, r2, cost = basic.cgls(Op, d, x0=x0, niter=FLOW_NITER, tol=0.0)
        return {"x": xinv.asarray(), "iiter": iiter, "cost": np.asarray(cost)}

    for P in (1, 2, 3):
        res = MPI.run_world(P, t_flow, P)[0]
        for k in ("x", "iiter", "cost"):
            out[f"flow/P{P}/{k}"] = np.asarray(res[k])
    spread = np.zeros(2)
    for seed in FLOW_JITTER_SEEDS:
        res = MPI.run_world(1, t_flow, 1, seed)[0]
        x1, c1 = out["flow/P1/x"], out["flow/P1/cost"]
        spread = np.maximum(spread, [np.abs(res["x"] - x1).max() / np.abs(x1).max(),
                                     (np.abs(res["cost"] - c1) / c1).max()])
    out["flow/spread"] = spread

    path = os.path.join(HERE, os.environ.get("GOLDEN_OUT", "nsconvolve3d_golden.npz"))
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1e3:.0f} KB, flow cond {float(out['flow/cond']):.3e}, "
          f"spread {out['flow/spread']}")


if __name__ == "__main__":
    main()
