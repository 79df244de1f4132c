"""Generate the non-stationary 2-D convolution fixtures by running the REAL reference's MPIBlockDiag and cgls (a
pylops-mpi checkout named by PYLOPS_MPI_REFERENCE, imported unmodified through make_golden.load_reference) over
refshim's restated ``pylops.signalprocessing.NonStationaryConvolve2D`` (refshim/pylops/signalprocessing/
nonstatconvolve2d.py) and, for the point-spread functions, refshim's ``pylops.waveeqprocessing.Kirchhoff``.

    PYLOPS_MPI_REFERENCE=<checkout> python tests/golden/make_golden_nsconvolve2d.py   # writes nsconvolve2d_golden.npz

Operator cases.  A (NY, NX, NZ) stack of images split along axis 0 over P in {1, 2, 3} ranks: rank r holds
MPIBlockDiag([NonStationaryConvolve2D((NX, NZ), hs_k, ihx, ihz) for its slices k]), one bank per slice.  Filter sizes
``NHS`` (1 x 1 to 41 x 41, square and not), banks ``BANKS`` (1 x 1, 2 x 3, 4 x 5 with steps 1 and 4 mixed over the
two axes), ihx = 1 + dhx * arange(nfx) and the same along z: both edges of both axes are extrapolated.  Inputs are
exactly representable: x has entries in {-1, 0, 1}, the taps are drawn from {-1, -1/2, 1/2, 1} and the steps are 1
or 4, so every bilinear weight is a multiple of 1/16, every output a multiple of 1/32, and each is the SAME in float64,
float32 and complex128 and at every P (all checked here).  Each output is stored once, losslessly, as int32 of
ENC * y.

  op/nh{nhx}x{nhz}/nf{nfx}x{nfz}/dh{dhx}x{dhz}/{y,ya}   gathered forward of x / adjoint of v
  .../{yi,yai}   imaginary parts of the complex128 runs, for the cases of ``complex_case``

Flow: image-domain least-squares migration.  A refshim Kirchhoff ``K`` (analytic, FLOW_NX x FLOW_NZ image) gives the
point-spread functions of a FLOW_NFX x FLOW_NFZ grid of point scatterers at (FLOW_IHX, FLOW_IHZ):
hs[a, b] = (K^H K m_psf)[px - hcx : px + hcx + 1, pz - hcz : pz + hcz + 1], and the migrated images
m_mig = K^H K m_true of FLOW_NY layered reflectivities.  Then cgls(MPIBlockDiag([NSC2D(hs)] * ny_r), m_mig, x0 = 0)
for FLOW_NITER iterations (tol = 0).

  flow/hs, flow/mmig, flow/P{P}/{x,iiter,cost}
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from fixture_codec import encode, rows_of  # noqa: E402

NY, NX, NZ = 4, 20, 24
NHS = ((1, 1), (3, 5), (7, 3), (1, 9), (41, 41))
BANKS = (((1, 1), (1, 1)), ((2, 3), (1, 4)), ((2, 3), (4, 1)), ((4, 5), (4, 4)), ((4, 5), (1, 1)))
DTYPES = ("float64", "float32", "complex128")
ENC = 32         # stored value = ENC * y, exact in int32

FLOW_NY, FLOW_NX, FLOW_NZ, FLOW_D = 4, 41, 31, 4.0
FLOW_NT, FLOW_DT, FLOW_VEL, FLOW_F0 = 151, 0.004, 1500.0, 25.0
FLOW_NH = (9, 9)
FLOW_IHX, FLOW_IHZ = (5, 15, 25, 35), (5, 15, 25)
FLOW_NITER = 20
REFSHIM = os.path.join(HERE, "refshim")


def complex_case(nh, bank):
    return nh == (3, 5) and bank[0] == (2, 3)


def cases():
    """(nh, (nf, dh), dtype)"""
    return [(nh, bank, dt) for nh in NHS for bank in BANKS for dt in DTYPES
            if dt != "complex128" or complex_case(nh, bank)]


def key(nh, bank):
    (nfx, nfz), (dhx, dhz) = bank
    return f"op/nh{nh[0]}x{nh[1]}/nf{nfx}x{nfz}/dh{dhx}x{dhz}"


def nodes(bank):
    """(ihx, ihz) of a bank: 1 + dh * arange(nf) per axis"""
    (nfx, nfz), (dhx, dhz) = bank
    return 1 + dhx * np.arange(nfx), 1 + dhz * np.arange(nfz)


def case_inputs(nh, bank, dt):
    """NY banks (the real dtype of dt), ihx, ihz, and the global x / v in dtype dt"""
    nf = bank[0]
    rng = np.random.default_rng(500 + 97 * nh[0] + 13 * nh[1] + 7 * nf[0] + nf[1] + bank[1][0])
    hs = rng.choice([-1.0, -0.5, 0.5, 1.0], (NY,) + nf + nh).astype(np.real(np.ones(1, dt)).dtype)
    ihx, ihz = nodes(bank)
    rng = np.random.default_rng(23)
    n = NY * NX * NZ
    x, v, xi, vi = (rng.integers(-1, 2, n).astype(np.float64) for _ in range(4))
    if dt == "complex128":
        x, v = x + 1j * xi, v + 1j * vi
    return hs, ihx, ihz, x.astype(dt), v.astype(dt)


def refshim_kirchhoff():
    added = REFSHIM not in sys.path
    if added:
        sys.path.insert(0, REFSHIM)
    try:
        import pylops.utils.wavelets as wavelets
        import pylops.waveeqprocessing.kirchhoff as kirchhoff
    finally:
        if added:
            sys.path.remove(REFSHIM)
    return kirchhoff, wavelets


def flow_geometry():
    """z, x, t, srcs, recs, vel, wav, wavc of the Kirchhoff operator whose K^H K the flow inverts"""
    _, wavelets = refshim_kirchhoff()
    x, z = np.arange(FLOW_NX) * FLOW_D, np.arange(FLOW_NZ) * FLOW_D
    t = np.arange(FLOW_NT) * FLOW_DT
    recs = np.vstack((np.linspace(0, x[-1], 21), np.zeros(21)))
    srcs = np.vstack((np.linspace(x[0] + 10 * FLOW_D, x[-1] - 10 * FLOW_D, 3), np.zeros(3)))
    wav, _, wavc = wavelets.ricker(t[:21], f0=FLOW_F0)
    return z, x, t, srcs, recs, FLOW_VEL, wav, int(wavc)


def flow_models():
    """(m_psf, m_true): the point scatterers at the filter nodes, and FLOW_NY layered reflectivities"""
    m_psf = np.zeros((FLOW_NX, FLOW_NZ))
    for px in FLOW_IHX:
        for pz in FLOW_IHZ:
            m_psf[px, pz] = 1.0
    m_true = np.zeros((FLOW_NY, FLOW_NX, FLOW_NZ))
    for k in range(FLOW_NY):
        m_true[k, :, 8 + k] = -1.0
        m_true[k, :, 20 - k] = 0.5
        m_true[k, 10 + 4 * k:16 + 4 * k, 14] = 0.75
    return m_psf, m_true


def psf_windows(m_psf_image):
    """hs[a, b] = the FLOW_NH window of K^H K m_psf around node (FLOW_IHX[a], FLOW_IHZ[b])"""
    hcx, hcz = FLOW_NH[0] // 2, FLOW_NH[1] // 2
    hs = np.zeros((len(FLOW_IHX), len(FLOW_IHZ)) + FLOW_NH)
    for a, px in enumerate(FLOW_IHX):
        for b, pz in enumerate(FLOW_IHZ):
            hs[a, b] = m_psf_image[px - hcx:px + hcx + 1, pz - hcz:pz + hcz + 1]
    return hs


def main():
    from make_golden import load_reference          # puts refshim/ (mpi4py, pylops) on the path
    from mpi4py import MPI
    from pylops.signalprocessing.nonstatconvolve2d import NonStationaryConvolve2D
    pkg, mods = load_reference()
    import importlib
    basic = importlib.import_module("pylops_mpi.optimization.basic")
    DA = pkg.DistributedArray
    BD = mods["BlockDiag"].MPIBlockDiag
    out = {}

    def t_op(rank, P, nh, bank, dt):
        hs, ihx, ihz, x, v = case_inputs(nh, bank, dt)
        ny = rows_of(P, NY)
        k0 = sum(ny[:rank])
        ls = [(r * NX * NZ,) for r in ny]
        Op = BD([NonStationaryConvolve2D((NX, NZ), hs[k], ihx, ihz, dtype=dt) for k in range(k0, k0 + ny[rank])],
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
                    for n in ("y", "ya"):                  # one bank per slice: the result does not depend on P
                        assert np.array_equal(res[n], runs[dt][n])
            k = key(nh, bank)
            for n in ("y", "ya"):
                assert np.array_equal(runs["float32"][n], runs["float64"][n])
                out[f"{k}/{n}"] = encode(runs["float64"][n], ENC, np.int32)
                if "complex128" in runs:
                    assert np.array_equal(runs["complex128"][n].real, runs["float64"][n])
                    out[f"{k}/{n}i"] = encode(runs["complex128"][n].imag, ENC, np.int32)

    # flow: the PSF bank and the migrated images from the restated Kirchhoff, in float64
    kirchhoff, _ = refshim_kirchhoff()
    z, x, t, srcs, recs, vel, wav, wavc = flow_geometry()
    K = kirchhoff.Kirchhoff(z, x, t, srcs, recs, vel, wav, wavc, mode="analytic")
    m_psf, m_true = flow_models()
    hs = psf_windows(K.rmatvec(K.matvec(m_psf.ravel())).reshape(FLOW_NX, FLOW_NZ))
    mmig = np.stack([K.rmatvec(K.matvec(m.ravel())) for m in m_true]).ravel()
    out["flow/hs"], out["flow/mmig"] = hs, mmig

    def t_flow(rank, P):
        ny = rows_of(P, FLOW_NY)
        ls = [(r * FLOW_NX * FLOW_NZ,) for r in ny]
        Op = BD([NonStationaryConvolve2D((FLOW_NX, FLOW_NZ), hs, FLOW_IHX, FLOW_IHZ)] * ny[rank])
        d = DA.to_dist(mmig, local_shapes=ls)
        x0 = DA(global_shape=mmig.size, local_shapes=ls)
        x0[:] = 0
        xinv, istop, iiter, r1, r2, cost = basic.cgls(Op, d, x0=x0, niter=FLOW_NITER, tol=0.0)
        return {"x": xinv.asarray(), "iiter": iiter, "cost": np.asarray(cost)}

    for P in (1, 2, 3):
        res = MPI.run_world(P, t_flow, P)[0]
        for k in ("x", "iiter", "cost"):
            out[f"flow/P{P}/{k}"] = np.asarray(res[k])

    path = os.path.join(HERE, os.environ.get("GOLDEN_OUT", "nsconvolve2d_golden.npz"))
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1e3:.0f} KB")


if __name__ == "__main__":
    main()
