"""Generate the Convolve1D fixtures by running the REAL reference's MPIBlockDiag and ISTA solver (a pylops-mpi
checkout named by PYLOPS_MPI_REFERENCE, imported unmodified through make_golden.load_reference) over refshim's restated
``pylops.signalprocessing.Convolve1D`` and ``pylops.FirstDerivative``.

    PYLOPS_MPI_REFERENCE=<checkout> python tests/golden/make_golden_convolve.py   # writes tests/golden/convolve_golden.npz

Inputs are exactly representable: x has entries in {-1, 0, 1} and the taps are drawn from {-1, -1/2, 1/2, 1}, so
every reference output is a multiple of 1/2 below 64 in magnitude and is the SAME in float64, float32 and complex128
(checked here).  Each output is therefore stored once, losslessly, as int8 of ENC * y.

  conv/P{P}/ax{axis}/nh{nh}/o{offset}/{y,ya}    gathered forward of x / adjoint of v through MPIBlockDiag([Convolve1D])
      on the global (7, 9, 33) array split along axis 0 (rank r owns a (ny_r, 9, 33) block), P in {1, 2, 3}; the
      float64, float32 and complex128 (real part) runs all equal it.  Axes -1 and 1 give the same result at every P
      and are stored once, as P "any" (see ``key``)
  conv/.../{yi,yai}  imaginary parts of the complex128 runs (x + 1j xi, v + 1j vi), for the cases of ``complex_case``
  refl/d, refl/alpha, refl/P{P}/{x,iiter,cost}  the reflectivity flow of tutorials/reflectivity.py on a (5, 4, 33)
      block split along axis 0: a blocky model, MPIBlockDiag([FirstDerivative(axis=-1)]) -> reflectivity, MPIBlockDiag([Convolve1D]) -> data d
      (bit-identical for every P), then 30 iterations of the ISTA class (what ``ista`` runs) with an explicit alpha
      (the reference's power iteration draws from a shared RNG).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from fixture_codec import encode, rows_of  # noqa: E402

DIMS = (7, 9, 33)
AXES = (-1, 0, 1)
NHS = (1, 5, 8, 41)
DTYPES = ("float64", "float32", "complex128")
REFL_DIMS, REFL_NH, REFL_OFF, REFL_EPS, REFL_NITER = (5, 4, 33), 15, 7, 0.05, 30


ENC = 2          # stored value = ENC * y, exact in int8


def offsets(nh):
    return sorted({0, nh // 2, nh - 1})


def complex_case(nh, off):
    return nh in (5, 41) and off == nh // 2


def cases():
    """(P, axis, nh, offset, dtype) of the operator tests: every combination in float64 / float32; complex128 at the
    middle offset of nh 5 and 41"""
    out = []
    for P in (1, 2, 3):
        for axis in AXES:
            for nh in NHS:
                for off in offsets(nh):
                    for dt in DTYPES:
                        if dt != "complex128" or complex_case(nh, off):
                            out.append((P, axis, nh, off, dt))
    return out


def key(P, axis, nh, off):
    """fixture key of one case: along axis -1 or 1 every rank convolves whole lines of its own rows, so the gathered
    result does not depend on P (checked when the fixture is made) and is stored once, under P "any" """
    return f"conv/P{P if along_rows(axis) else 'any'}/ax{axis}/nh{nh}/o{off}"


def along_rows(axis):
    """does the convolution run along axis 0, the one split across ranks?"""
    return axis % len(DIMS) == 0


def case_inputs(nh, dt):
    """taps h (float64) and the global x (forward input) and v (adjoint input) of one case, in dtype dt"""
    h = np.random.default_rng(100 + nh).choice([-1.0, -0.5, 0.5, 1.0], nh)
    rng = np.random.default_rng(7)
    n = int(np.prod(DIMS))
    x, v, xi, vi = (rng.integers(-1, 2, n).astype(np.float64) for _ in range(4))
    if dt == "complex128":
        x, v = x + 1j * xi, v + 1j * vi
    return h, x.astype(dt), v.astype(dt)


def refl_inputs():
    """wavelet (Ricker, 15 taps, centred), blocky model, ista step"""
    t = (np.arange(REFL_NH) - REFL_OFF) * 0.004
    f0 = 20.0
    wav = (1 - 2 * (np.pi * f0 * t) ** 2) * np.exp(-(np.pi * f0 * t) ** 2)
    rng = np.random.default_rng(11)
    m = np.zeros(REFL_DIMS)
    for iy in range(REFL_DIMS[0]):
        for ix in range(REFL_DIMS[1]):
            cuts = np.sort(rng.choice(np.arange(2, REFL_DIMS[2] - 2), 4, replace=False))
            m[iy, ix] = np.repeat(rng.standard_normal(5), np.diff(np.r_[0, cuts, REFL_DIMS[2]]))
    alpha = 1.0 / float(np.sum(np.abs(wav)) ** 2)      # ||C|| <= ||h||_1
    return wav, m.ravel(), alpha


def main():
    from make_golden import load_reference          # puts refshim/ (mpi4py, pylops) on the path
    from mpi4py import MPI
    import pylops
    from pylops.signalprocessing.convolve1d import Convolve1D
    pkg, mods = load_reference()
    DA = pkg.DistributedArray
    BD = mods["BlockDiag"].MPIBlockDiag
    ISTA = mods["cls_sparsity"].ISTA
    out = {}

    def t_conv(rank, P, axis, nh, off, dt):
        h, x, v = case_inputs(nh, dt)
        ny = rows_of(P, DIMS[0])
        ls = [(r * DIMS[1] * DIMS[2],) for r in ny]
        Op = BD([Convolve1D((ny[rank],) + DIMS[1:], h, offset=off, axis=axis, dtype=dt)])
        fwd = Op @ DA.to_dist(x, local_shapes=ls)
        adj = Op.H @ DA.to_dist(v, local_shapes=ls)
        return {"y": fwd.asarray(), "ya": adj.asarray()}

    for P in (1, 2, 3):
        for axis in AXES:
            for nh in NHS:
                for off in offsets(nh):
                    runs = {}
                    for dt in DTYPES:
                        if dt == "complex128" and not complex_case(nh, off):
                            continue
                        res = MPI.run_world(P, t_conv, P, axis, nh, off, dt)
                        for r in range(1, P):
                            assert all(np.array_equal(res[r][n], res[0][n]) for n in ("y", "ya"))
                        runs[dt] = res[0]
                    k = key(P, axis, nh, off)
                    enc = {}
                    for n in ("y", "ya"):
                        enc[n] = encode(runs["float64"][n], ENC, np.int8)
                        assert np.array_equal(runs["float32"][n], runs["float64"][n])
                        if "complex128" in runs:
                            assert np.array_equal(runs["complex128"][n].real, runs["float64"][n])
                            enc[f"{n}i"] = encode(runs["complex128"][n].imag, ENC, np.int8)
                    for n, e in enc.items():
                        if f"{k}/{n}" in out:                   # P-independent case, stored at P = 1
                            assert np.array_equal(out[f"{k}/{n}"], e)
                        else:
                            out[f"{k}/{n}"] = e

    def t_refl(rank, P):
        wav, m, alpha = refl_inputs()
        ny = rows_of(P, REFL_DIMS[0])
        ls = [(r * REFL_DIMS[1] * REFL_DIMS[2],) for r in ny]
        dims = (ny[rank],) + REFL_DIMS[1:]
        DDiag = BD([pylops.FirstDerivative(dims, axis=-1)])
        CDiag = BD([Convolve1D(dims, wav, offset=REFL_OFF, axis=-1)])
        r = DDiag @ DA.to_dist(m, local_shapes=ls)
        d = CDiag @ r
        x0 = DA(global_shape=m.size, local_shapes=ls)
        x0[:] = 0
        x, iiter, cost = ISTA(CDiag).solve(d, x0, niter=REFL_NITER, eps=REFL_EPS, alpha=alpha, tol=1e-10)
        return {"x": x.asarray(), "iiter": iiter, "cost": np.asarray(cost), "alpha": alpha, "d": d.asarray()}

    for P in (1, 2, 3):
        res = MPI.run_world(P, t_refl, P)[0]
        if P == 1:
            out["refl/d"], out["refl/alpha"] = res["d"], np.asarray(res["alpha"])
        assert np.array_equal(res["d"], out["refl/d"])
        for k in ("x", "iiter", "cost"):
            out[f"refl/P{P}/{k}"] = np.asarray(res[k])

    path = os.path.join(HERE, os.environ.get("GOLDEN_OUT", "convolve_golden.npz"))
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
