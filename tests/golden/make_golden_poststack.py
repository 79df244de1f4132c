"""Generate the PoststackLinearModelling fixtures by running the REAL reference's MPIBlockDiag, cgls / CGLS, cg,
MPILaplacian and MPIStackedVStack (a pylops-mpi checkout named by PYLOPS_MPI_REFERENCE, imported unmodified through
make_golden.load_reference) over refshim's restated ``pylops.avo.poststack.PoststackLinearModelling``,
``pylops.basicoperators.Transpose`` (refshim/pylops/basicoperators/transpose.py) and their operator products
(refshim/pylops/_algebra.py).

    PYLOPS_MPI_REFERENCE=<checkout> python tests/golden/make_golden_poststack.py   # writes tests/golden/poststack_golden.npz

Operator cases.  Inputs are exactly representable: x has entries in {-1, 0, 1} and the wavelet taps are drawn from
{-1, -1/2, 1/2, 1}, so every reference output is a multiple of 1/4 and is the SAME in float64, float32 and
complex128 (checked here).  Each output is stored once, losslessly, as int16 of ENC * y (|y| exceeds 127 / ENC at
nh = 41).

  op/{layout}/P{P}/{kind}/nh{nh}/{y,ya}   gathered forward of x / adjoint of v through MPIBlockDiag at P in {1, 2, 3}
      layout "native": rank r owns a (NT0, ny_r, NX) block, operator PoststackLinearModelling(wav, NT0, (ny_r, NX))
      layout "tut":    rank r owns a (ny_r, NX, NT0) block, operator Top.H @ PPop @ Top as in tutorials/poststack.py
                       (time runs along whole lines inside each rank's rows: the result does not depend on P and is
                       stored once, as P "any")
  op/.../{yi,yai}  imaginary parts of the complex128 runs (x + 1j xi, v + 1j vi), for the cases of ``complex_case``
  flow/d, flow/P{P}/{iter,ne,reg}/{x,iiter,cost}  the three solves of tutorials/poststack.py on a (FLOW_NY, NX, NT0)
      blocky log-impedance model split along y, with a restated 15-tap Ricker wavelet (float64): the modelled data d
      (identical at every P), FLOW_NITER iterations of cgls from a smoothed model, of cg on the normal equations
      BDiag.H @ BDiag + epsR * LapOp.H @ LapOp, and of cgls on MPIStackedVStack([BDiag, sqrt(epsR) * LapOp]).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from fixture_codec import encode, rows_of  # noqa: E402

NY, NX, NT0 = 5, 4, 33
LAYOUTS = ("native", "tut")
KINDS = ("centered", "forward")
NHS = (1, 4, 5, 41)
DTYPES = ("float64", "float32", "complex128")
ENC = 4          # stored value = ENC * y, exact in int16
FLOW_NWAV, FLOW_F0, FLOW_DT, FLOW_EPSR, FLOW_NITER = 15, 15.0, 0.004, 1e2, 10
FLOW_NY = 6      # the reference's MPILaplacian needs at least 2 rows of y on every rank (P = 3)


def complex_case(layout, kind, nh):
    return kind == "centered" and nh == 5


def cases():
    """(layout, P, kind, nh, dtype) of the operator tests: every combination in float64 / float32; complex128 at the
    centered nh = 5 cases"""
    return [(layout, P, kind, nh, dt) for layout in LAYOUTS for P in (1, 2, 3) for kind in KINDS for nh in NHS
            for dt in DTYPES if dt != "complex128" or complex_case(layout, kind, nh)]


def block_dims(layout, ny_r):
    return (NT0, ny_r, NX) if layout == "native" else (ny_r, NX, NT0)


def key(layout, P, kind, nh):
    return f"op/{layout}/P{P if layout == 'native' else 'any'}/{kind}/nh{nh}"


def case_inputs(nh, dt):
    """wavelet and the global x (forward input) and v (adjoint input) of one case: x and v in dtype dt, the wavelet
    (whose dtype is the operator's) in the real dtype of dt.  MPIBlockDiag is built with dtype dt, so that complex
    data keep their imaginary part"""
    wav = np.random.default_rng(200 + nh).choice([-1.0, -0.5, 0.5, 1.0], nh).astype(np.real(np.ones(1, dt)).dtype)
    rng = np.random.default_rng(17)
    n = NY * NX * NT0
    x, v, xi, vi = (rng.integers(-1, 2, n).astype(np.float64) for _ in range(4))
    if dt == "complex128":
        x, v = x + 1j * xi, v + 1j * vi
    return wav, x.astype(dt), v.astype(dt)


def ricker(t, f0):
    """pylops.utils.wavelets.ricker restated: the symmetric Ricker wavelet on [-t[-1], t[-1]]"""
    w = (1 - 2 * (np.pi * f0 * t) ** 2) * np.exp(-(np.pi * f0 * t) ** 2)
    return np.concatenate((np.flipud(w[1:]), w), axis=0)


def smooth(a, n, axis):
    """zero-phase moving average (scipy.signal.filtfilt of a box filter), as tutorials/poststack.py smooths"""
    from scipy.signal import filtfilt
    return filtfilt(np.ones(n) / float(n), 1, a, axis=axis)


def flow_inputs():
    """wavelet, global log-impedance model m3d (FLOW_NY, NX, NT0) and its smoothed background mback3d"""
    wav = ricker(np.arange(FLOW_NWAV // 2 + 1) * FLOW_DT, FLOW_F0)
    rng = np.random.default_rng(23)
    prof = np.zeros((NX, NT0))
    for ix in range(NX):
        cuts = np.sort(rng.choice(np.arange(3, NT0 - 3), 4, replace=False))
        prof[ix] = np.log(np.repeat(2000 + 1500 * rng.random(5), np.diff(np.r_[0, cuts, NT0])))
    m3d = np.tile(prof[np.newaxis], (FLOW_NY, 1, 1)) + 0.01 * rng.standard_normal((FLOW_NY, NX, NT0))
    mback3d = smooth(m3d, 7, 2)          # along time only: y and x are shorter than filtfilt's padding
    return wav, m3d, mback3d


def main():
    from make_golden import load_reference          # puts refshim/ (mpi4py, pylops) on the path
    from mpi4py import MPI
    from pylops.avo.poststack import PoststackLinearModelling
    from pylops.basicoperators.transpose import Transpose
    pkg, mods = load_reference()
    import importlib
    basic = importlib.import_module("pylops_mpi.optimization.basic")
    DA, SDA = pkg.DistributedArray, pkg.StackedDistributedArray
    BD = mods["BlockDiag"].MPIBlockDiag
    SVS = mods["VStack"].MPIStackedVStack
    LAP = mods["Laplacian"].MPILaplacian
    out = {}

    def local_op(layout, ny_r, wav, kind):
        if layout == "native":
            return PoststackLinearModelling(wav, nt0=NT0, spatdims=(ny_r, NX), kind=kind)
        PPop = PoststackLinearModelling(wav, nt0=NT0, spatdims=(ny_r, NX), kind=kind)
        Top = Transpose((ny_r, NX, NT0), (2, 0, 1))
        return Top.H @ PPop @ Top

    def t_op(rank, layout, P, kind, nh, dt):
        wav, x, v = case_inputs(nh, dt)
        ny = rows_of(P, NY)
        ls = [(r * NX * NT0,) for r in ny]
        Op = BD([local_op(layout, ny[rank], wav, kind)], dtype=dt)
        fwd = Op @ DA.to_dist(x, local_shapes=ls)
        adj = Op.H @ DA.to_dist(v, local_shapes=ls)
        return {"y": fwd.asarray(), "ya": adj.asarray()}

    for layout in LAYOUTS:
        for P in (1, 2, 3):
            for kind in KINDS:
                for nh in NHS:
                    runs = {}
                    for dt in DTYPES:
                        if dt == "complex128" and not complex_case(layout, kind, nh):
                            continue
                        res = MPI.run_world(P, t_op, layout, P, kind, nh, dt)
                        runs[dt] = res[0]
                    k = key(layout, P, kind, nh)
                    enc = {}
                    for n in ("y", "ya"):
                        enc[n] = encode(runs["float64"][n], ENC, np.int16)
                        assert np.array_equal(runs["float32"][n], runs["float64"][n])
                        if "complex128" in runs:
                            assert np.array_equal(runs["complex128"][n].real, runs["float64"][n])
                            enc[f"{n}i"] = encode(runs["complex128"][n].imag, ENC, np.int16)
                    for n, e in enc.items():
                        if f"{k}/{n}" in out:                   # P-independent case, stored at P = 1
                            assert np.array_equal(out[f"{k}/{n}"], e)
                        else:
                            out[f"{k}/{n}"] = e

    def t_flow(rank, P):
        """tutorials/poststack.py at (NY, NX, NT0), y split over P ranks"""
        wav, m3d, mback3d = flow_inputs()
        ny = rows_of(P, FLOW_NY)
        y0 = sum(ny[:rank])
        ny_i = ny[rank]
        ls = [(r * NX * NT0,) for r in ny]
        m3d_dist = DA(global_shape=FLOW_NY * NX * NT0, local_shapes=ls)
        m3d_dist[:] = m3d[y0:y0 + ny_i].flatten()
        mback3d_dist = DA(global_shape=FLOW_NY * NX * NT0, local_shapes=ls)
        mback3d_dist[:] = mback3d[y0:y0 + ny_i].flatten()
        PPop = PoststackLinearModelling(wav, nt0=NT0, spatdims=(ny_i, NX))
        Top = Transpose((ny_i, NX, NT0), (2, 0, 1))
        BDiag = BD(ops=[Top.H @ PPop @ Top, ])
        d_dist = BDiag @ m3d_dist
        res = {"d": d_dist.asarray()}
        x, istop, iiter, r1, r2, cost = basic.cgls(BDiag, d_dist, x0=mback3d_dist, niter=FLOW_NITER, tol=0.0)
        res["iter"] = (x.asarray(), iiter, cost)
        LapOp = LAP(dims=(FLOW_NY, NX, NT0), axes=(0, 1, 2), weights=(1, 1, 1), sampling=(1, 1, 1), dtype=BDiag.dtype)
        NormEqOp = BDiag.H @ BDiag + FLOW_EPSR * LapOp.H @ LapOp
        dnorm_dist = BDiag.H @ d_dist
        x, iiter, cost = basic.cg(NormEqOp, dnorm_dist, x0=mback3d_dist, niter=FLOW_NITER, tol=0.0)
        res["ne"] = (x.asarray(), iiter, cost)
        StackOp = SVS([BDiag, np.sqrt(FLOW_EPSR) * LapOp])
        d0_dist = DA(global_shape=FLOW_NY * NX * NT0, local_shapes=ls)
        d0_dist[:] = 0.
        dstack_dist = SDA([d_dist, d0_dist])
        x, istop, iiter, r1, r2, cost = basic.cgls(StackOp, dstack_dist, x0=mback3d_dist, niter=FLOW_NITER, tol=0.0)
        res["reg"] = (x.asarray(), iiter, cost)
        return res

    for P in (1, 2, 3):
        res = MPI.run_world(P, t_flow, P)[0]
        if P == 1:
            out["flow/d"] = res["d"]
        assert np.array_equal(res["d"], out["flow/d"])
        for name in ("iter", "ne", "reg"):
            x, iiter, cost = res[name]
            out[f"flow/P{P}/{name}/x"] = np.asarray(x)
            out[f"flow/P{P}/{name}/iiter"] = np.asarray(iiter)
            out[f"flow/P{P}/{name}/cost"] = np.asarray(cost)

    path = os.path.join(HERE, os.environ.get("GOLDEN_OUT", "poststack_golden.npz"))
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
