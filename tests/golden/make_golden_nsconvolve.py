"""Generate the non-stationary convolution fixtures by running the REAL reference's MPIBlockDiag, cgls and ISTA (a
pylops-mpi checkout named by PYLOPS_MPI_REFERENCE, imported unmodified through make_golden.load_reference) over
refshim's restated ``pylops.signalprocessing.NonStationaryConvolve1D`` and the 2-D wavelet branch of
``pylops.avo.poststack.PoststackLinearModelling`` (refshim/pylops/avo/poststack_nonstationary.py:
``nonstationary_convmtx`` through ``MatrixMult`` with ``otherdims``).

    PYLOPS_MPI_REFERENCE=<checkout> python tests/golden/make_golden_nsconvolve.py   # writes tests/golden/nsconvolve_golden.npz

Operator cases.  Inputs are exactly representable: x has entries in {-1, 0, 1}, the taps are drawn from
{-1, -1/2, 1/2, 1} and the filter spacing dh is 1 or 4, so every interpolated tap and every output is a multiple of
1/8 and is the SAME in float64, float32 and complex128 (checked here).  Each output is stored once, losslessly, as
int16 of ENC * y.

  ns/P{P}/ax{axis}/nh{nh}/nf{nfilt}/dh{dh}/{y,ya}   NonStationaryConvolve1D(dims, hs, ih, axis) on the global DIMS
      array split along axis 0 (rank r owns a (ny_r,) + DIMS[1:] block), ih = 1 + dh * arange(nfilt): both ends of the
      axis are extrapolated.  Axis -1 does not depend on P and is stored once, as P "any"
  post/{layout}/P{P}/{kind}/nw{nwav}/{y,ya}   PoststackLinearModelling(wav (NT0, nwav), NT0, (ny_r, NX), kind), in
      the "native" (NT0, ny_r, NX) and "tut" (Top.H @ PPop @ Top on (ny_r, NX, NT0)) layouts of
      make_golden_poststack.py; "tut" is stored once, as P "any"
  .../{yi,yai}   imaginary parts of the complex128 runs, for the cases of ``complex_ns`` / ``complex_post``
  flow/d, flow/P{P}/{x,iiter,cost}   tutorials/poststack.py's cgls on a (FLOW_NY, NX, NT0) model with a Ricker
      wavelet whose peak frequency falls with time (one wavelet per sample)
  ista/d, ista/alpha, ista/P{P}/{x,iiter,cost}   ISTA on MPIBlockDiag([NonStationaryConvolve1D(axis=-1)])
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from fixture_codec import encode, rows_of  # noqa: E402
import make_golden_poststack as mgp  # noqa: E402

DIMS = (60, 2, 24)
AXES = (-1, 0)
NHS = (1, 5, 41)
NFILTS = (1, 2, 5)
DHS = (1, 4)
NWAVS = (1, 4, 5, 41)
LAYOUTS, KINDS = mgp.LAYOUTS, mgp.KINDS
NY, NX, NT0 = mgp.NY, mgp.NX, mgp.NT0
DTYPES = ("float64", "float32", "complex128")
ENC = 8          # stored value = ENC * y, exact in int16
FLOW_NY, FLOW_NWAV, FLOW_DT, FLOW_F0, FLOW_NITER = mgp.FLOW_NY, 15, 0.004, (25.0, 10.0), 10
ISTA_DIMS, ISTA_NH, ISTA_IH, ISTA_EPS, ISTA_NITER = (5, 4, 40), 15, (4, 14, 24, 34), 0.05, 30


def complex_ns(nh, nfilt, dh):
    return nh == 5 and nfilt == 2 and dh == 4


def complex_post(kind, nwav):
    return kind == "centered" and nwav == 5


def ns_configs():
    """(nh, nfilt, dh); dh does not matter for one filter"""
    return [(nh, nf, dh) for nh in NHS for nf in NFILTS for dh in DHS if nf > 1 or dh == 1]


def ns_cases():
    return [(P, axis, nh, nf, dh, dt) for P in (1, 2, 3) for axis in AXES for nh, nf, dh in ns_configs()
            for dt in DTYPES if dt != "complex128" or complex_ns(nh, nf, dh)]


def post_cases():
    return [(layout, P, kind, nw, dt) for layout in LAYOUTS for P in (1, 2, 3) for kind in KINDS for nw in NWAVS
            for dt in DTYPES if dt != "complex128" or complex_post(kind, nw)]


def ns_key(P, axis, nh, nf, dh):
    return f"ns/P{P if axis == 0 else 'any'}/ax{axis}/nh{nh}/nf{nf}/dh{dh}"


def post_key(layout, P, kind, nw):
    return f"post/{layout}/P{P if layout == 'native' else 'any'}/{kind}/nw{nw}"


def taps(shape, seed):
    return np.random.default_rng(seed).choice([-1.0, -0.5, 0.5, 1.0], shape)


def ns_inputs(nh, nf, dh, dt):
    """filter bank (real dtype of dt), ih, and the global x / v in dtype dt"""
    hs = taps((nf, nh), 300 + 10 * nh + nf).astype(np.real(np.ones(1, dt)).dtype)
    ih = 1 + dh * np.arange(nf)
    rng = np.random.default_rng(19)
    n = int(np.prod(DIMS))
    x, v, xi, vi = (rng.integers(-1, 2, n).astype(np.float64) for _ in range(4))
    if dt == "complex128":
        x, v = x + 1j * xi, v + 1j * vi
    return hs, ih, x.astype(dt), v.astype(dt)


def post_inputs(nw, dt):
    """2-D wavelet (NT0, nw) in the real dtype of dt, and the global x / v in dtype dt"""
    wav = taps((NT0, nw), 400 + nw).astype(np.real(np.ones(1, dt)).dtype)
    _, x, v = mgp.case_inputs(1, dt)
    return wav, x, v


def ricker(t, f0):
    w = (1 - 2 * (np.pi * f0 * t) ** 2) * np.exp(-(np.pi * f0 * t) ** 2)
    return np.concatenate((np.flipud(w[1:]), w), axis=0)


def flow_inputs():
    """time-varying Ricker wavelets (NT0, FLOW_NWAV), peak frequency falling linearly with time; model, background"""
    t = np.arange(FLOW_NWAV // 2 + 1) * FLOW_DT
    f0 = np.linspace(FLOW_F0[0], FLOW_F0[1], NT0)
    wav = np.stack([ricker(t, f) for f in f0])
    _, m3d, mback3d = mgp.flow_inputs()
    return wav, m3d, mback3d


def ista_inputs():
    """filter bank (Ricker wavelets, falling frequency), blocky model, ista step"""
    t = (np.arange(ISTA_NH) - ISTA_NH // 2) * 0.004
    hs = np.stack([(1 - 2 * (np.pi * f * t) ** 2) * np.exp(-(np.pi * f * t) ** 2) for f in (30.0, 24.0, 18.0, 12.0)])
    rng = np.random.default_rng(29)
    m = np.zeros(ISTA_DIMS)
    for iy in range(ISTA_DIMS[0]):
        for ix in range(ISTA_DIMS[1]):
            cuts = np.sort(rng.choice(np.arange(2, ISTA_DIMS[2] - 2), 4, replace=False))
            m[iy, ix] = np.repeat(rng.standard_normal(5), np.diff(np.r_[0, cuts, ISTA_DIMS[2]]))
    alpha = 1.0 / float(np.abs(hs).sum(axis=1).max() ** 2)      # every row and column of C has |.|_1 <= max |h|_1
    return hs, np.asarray(ISTA_IH), m.ravel(), alpha


def main():
    from make_golden import load_reference          # puts refshim/ (mpi4py, pylops) on the path
    from mpi4py import MPI
    from pylops.avo.poststack_nonstationary import PoststackLinearModelling
    from pylops.basicoperators.transpose import Transpose
    from pylops.signalprocessing.nonstatconvolve1d import NonStationaryConvolve1D
    pkg, mods = load_reference()
    import importlib
    basic = importlib.import_module("pylops_mpi.optimization.basic")
    DA = pkg.DistributedArray
    BD = mods["BlockDiag"].MPIBlockDiag
    ISTA = mods["cls_sparsity"].ISTA
    out = {}

    def store(k, runs):
        enc = {}
        for n in ("y", "ya"):
            enc[n] = encode(runs["float64"][n], ENC, np.int16)
            assert np.array_equal(runs["float32"][n], runs["float64"][n])
            if "complex128" in runs:
                assert np.array_equal(runs["complex128"][n].real, runs["float64"][n])
                enc[f"{n}i"] = encode(runs["complex128"][n].imag, ENC, np.int16)
        for n, e in enc.items():
            if f"{k}/{n}" in out:                       # P-independent case, stored at P = 1
                assert np.array_equal(out[f"{k}/{n}"], e)
            else:
                out[f"{k}/{n}"] = e

    def t_ns(rank, P, axis, nh, nf, dh, dt):
        hs, ih, x, v = ns_inputs(nh, nf, dh, dt)
        ny = rows_of(P, DIMS[0])
        ls = [(r * DIMS[1] * DIMS[2],) for r in ny]
        Op = BD([NonStationaryConvolve1D((ny[rank],) + DIMS[1:], hs, ih, axis=axis, dtype=dt)], dtype=dt)
        return {"y": (Op @ DA.to_dist(x, local_shapes=ls)).asarray(),
                "ya": (Op.H @ DA.to_dist(v, local_shapes=ls)).asarray()}

    for P in (1, 2, 3):
        for axis in AXES:
            for nh, nf, dh in ns_configs():
                runs = {dt: MPI.run_world(P, t_ns, P, axis, nh, nf, dh, dt)[0] for dt in DTYPES
                        if dt != "complex128" or complex_ns(nh, nf, dh)}
                store(ns_key(P, axis, nh, nf, dh), runs)

    def local_post(layout, ny_r, wav, kind):
        PPop = PoststackLinearModelling(wav, nt0=NT0, spatdims=(ny_r, NX), kind=kind)
        if layout == "native":
            return PPop
        Top = Transpose((ny_r, NX, NT0), (2, 0, 1))
        return Top.H @ PPop @ Top

    def t_post(rank, layout, P, kind, nw, dt):
        wav, x, v = post_inputs(nw, dt)
        ny = rows_of(P, mgp.NY)
        ls = [(r * NX * NT0,) for r in ny]
        Op = BD([local_post(layout, ny[rank], wav, kind)], dtype=dt)
        return {"y": (Op @ DA.to_dist(x, local_shapes=ls)).asarray(),
                "ya": (Op.H @ DA.to_dist(v, local_shapes=ls)).asarray()}

    for layout in LAYOUTS:
        for P in (1, 2, 3):
            for kind in KINDS:
                for nw in NWAVS:
                    runs = {dt: MPI.run_world(P, t_post, layout, P, kind, nw, dt)[0] for dt in DTYPES
                            if dt != "complex128" or complex_post(kind, nw)}
                    store(post_key(layout, P, kind, nw), runs)

    def t_flow(rank, P):
        """tutorials/poststack.py's modelling and cgls, with one wavelet per time sample"""
        wav, m3d, mback3d = flow_inputs()
        ny = rows_of(P, FLOW_NY)
        y0, ny_i = sum(ny[:rank]), ny[rank]
        ls = [(r * NX * NT0,) for r in ny]
        m3d_dist = DA(global_shape=FLOW_NY * NX * NT0, local_shapes=ls)
        m3d_dist[:] = m3d[y0:y0 + ny_i].flatten()
        mback3d_dist = DA(global_shape=FLOW_NY * NX * NT0, local_shapes=ls)
        mback3d_dist[:] = mback3d[y0:y0 + ny_i].flatten()
        PPop = PoststackLinearModelling(wav, nt0=NT0, spatdims=(ny_i, NX))
        Top = Transpose((ny_i, NX, NT0), (2, 0, 1))
        BDiag = BD(ops=[Top.H @ PPop @ Top, ])
        d_dist = BDiag @ m3d_dist
        x, istop, iiter, r1, r2, cost = basic.cgls(BDiag, d_dist, x0=mback3d_dist, niter=FLOW_NITER, tol=0.0)
        return {"d": d_dist.asarray(), "x": x.asarray(), "iiter": iiter, "cost": np.asarray(cost)}

    def t_ista(rank, P):
        hs, ih, m, alpha = ista_inputs()
        ny = rows_of(P, ISTA_DIMS[0])
        ls = [(r * ISTA_DIMS[1] * ISTA_DIMS[2],) for r in ny]
        CDiag = BD([NonStationaryConvolve1D((ny[rank],) + ISTA_DIMS[1:], hs, ih, axis=-1)])
        d = CDiag @ DA.to_dist(m, local_shapes=ls)
        x0 = DA(global_shape=m.size, local_shapes=ls)
        x0[:] = 0
        x, iiter, cost = ISTA(CDiag).solve(d, x0, niter=ISTA_NITER, eps=ISTA_EPS, alpha=alpha, tol=1e-10)
        return {"d": d.asarray(), "x": x.asarray(), "iiter": iiter, "cost": np.asarray(cost), "alpha": alpha}

    for name, fn in (("flow", t_flow), ("ista", t_ista)):
        for P in (1, 2, 3):
            res = MPI.run_world(P, fn, P)[0]
            if P == 1:
                out[f"{name}/d"] = res["d"]
                if name == "ista":
                    out["ista/alpha"] = np.asarray(res["alpha"])
            assert np.array_equal(res["d"], out[f"{name}/d"])
            for k in ("x", "iiter", "cost"):
                out[f"{name}/P{P}/{k}"] = np.asarray(res[k])

    path = os.path.join(HERE, os.environ.get("GOLDEN_OUT", "nsconvolve_golden.npz"))
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1e3:.0f} KB")


if __name__ == "__main__":
    main()
