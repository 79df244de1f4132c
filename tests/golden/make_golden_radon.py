"""Generate the Radon2D / Radon3D fixtures by running the REAL reference's MPIBlockDiag and FISTA (a pylops-mpi
checkout named by PYLOPS_MPI_REFERENCE, imported unmodified through make_golden.load_reference) over refshim's
restated ``pylops.signalprocessing.Radon2D`` / ``Radon3D`` (refshim/pylops/signalprocessing/radon2d.py, radon3d.py).

    PYLOPS_MPI_REFERENCE=<checkout> python tests/golden/make_golden_radon.py   # writes radon_golden.npz

NG gathers split over P in {1, 2, 3} ranks: rank r holds MPIBlockDiag([Radon(...) for each of its gathers], dtype),
float32 / float64 operators (float64 for complex data) and dtype the data's.  Every kind x interp x centeredh, in
2-D (NT2 = 37 samples, NH2 = 6 or 7 traces, 5 slownesses) and 3-D (NT3 = 19 samples, 3 x 4 traces, 2 x 3
slownesses).  dt = 2^-8 and dh = 8 (3-D: dhy = 16, dhx = 8), and the p axes are the unitless
values ``PU`` scaled back to physical units, so every unitless h and p is dyadic: h a multiple of 1/2, p of 1/8.
The p axes hold negative values, zero (a hyperbolic velocity of 0: every pair of that trace drops out) and slopes that
leave the trace at both ends; an odd centred gather has h = 0, where t0 = nt - 1 lands exactly on tdec = nt - 1.
Model x and data v have entries in {-1, 0, 1}.  Then every linear and parabolic d is a multiple of 1/32, and every
output of those kinds, and of the hyperbolic kind without interpolation, is a multiple of 1/64: the SAME in float64,
float32 and complex128 and at every P (all checked here), stored once, losslessly, as int32 of ENC * y.  Hyperbolic
curves with interpolation have irrational weights: their outputs are stored as the float64 run (the same bits at every
P, checked here) and the tests compare other dtypes and summation orders under a rounding bound.

  op/{2d,3d}/{kind}/i{interp}/c{centeredh}/{y,ya}     gathered forward of x / adjoint of v
  .../{yi,yai}   imaginary parts of the complex128 runs, for the cases of ``complex_case``

Flow: sparse linear-Radon denoising.  FLOW_NG synthetic CMP gathers of FLOW_NH traces and FLOW_NT samples, each a
few linear events (spikes in the Radon domain, seeded) plus seeded noise, split over the ranks; then FISTA (the class
``fista`` runs) on MPIBlockDiag([Radon2D(..., kind="linear")]), x0 = 0, FLOW_NITER iterations, sparsity FLOW_EPS and
the explicit step ``alpha`` = 1 / (||A||_1 ||A||_inf) of one gather's dense matrix (the reference's power iteration
draws from a shared RNG).  ``cond`` is that matrix's 2-norm condition number and ``spread`` how far rounding alone
moves the reference's own run: the largest change of x (relative to max |x|) and of the cost (relative) when every
apply of the restated operator is jittered by 4 ulps, over FLOW_JITTER_SEEDS at P = 1.  The tests take their
tolerance from both.

  flow/d, flow/m, flow/alpha, flow/cond, flow/spread, flow/P{P}/{x,iiter,cost}
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REFSHIM = os.path.join(HERE, "refshim")
sys.path.insert(0, HERE)
from fixture_codec import encode, rows_of  # noqa: E402

NG = 6
DT = 2.0 ** -8
DH2, DH3 = 8.0, (16.0, 8.0)
NT2, NH2 = 37, (6, 7)
NT3, NH3 = 19, (3, 4)
KINDS = ("linear", "parabolic", "hyperbolic")
# unitless slownesses (linear, parabolic) and velocities (hyperbolic) of the model traces
PU2 = {"linear": (-1.5, -0.75, 0.0, 0.5, 1.25), "parabolic": (-0.5, -0.125, 0.0, 0.25, 0.75),
       "hyperbolic": (0.0, 0.25, 0.5, 1.0, 2.0)}
PU3 = {"linear": ((-0.5, 0.75), (-1.25, 0.0, 0.5)), "parabolic": ((-0.25, 0.125), (-0.5, 0.0, 0.375)),
       "hyperbolic": ((0.5, 2.0), (0.0, 0.25, 1.0))}
DTYPES = ("float64", "float32", "complex128")
ENC = 64         # stored value = ENC * y, exact in int32

FLOW_NG, FLOW_NT, FLOW_NH, FLOW_NITER, FLOW_EPS = 6, 64, 16, 30, 0.1
FLOW_PU = tuple(np.arange(-2.0, 2.01, 0.25))          # 17 unitless slopes
FLOW_JITTER_SEEDS = (1, 2, 3)


def exact(kind, interp):
    """are the outputs of this kind exactly representable (dyadic weights, or no weights)?"""
    return kind != "hyperbolic" or not interp


def complex_case(kind, interp, centeredh):
    return exact(kind, interp) and centeredh


def cases():
    """(ndim, kind, interp, centeredh, nh) -- nh: 2-D the trace count, 3-D None; one entry per stored case"""
    out = []
    for kind in KINDS:
        for interp in (True, False):
            for centeredh in (True, False):
                for nh in NH2:
                    out.append((2, kind, interp, centeredh, nh))
                out.append((3, kind, interp, centeredh, None))
    return out


def key(ndim, kind, interp, centeredh, nh):
    return f"op/{ndim}d/{kind}/i{int(interp)}/c{int(centeredh)}" + (f"/nh{nh}" if ndim == 2 else "")


def haxis(nh, dh, centeredh):
    """physical offsets: centred gathers any origin (the operator recentres them), else traces -1 .. nh - 2"""
    return (np.arange(nh) - (nh // 2 if centeredh else 1)) * dh


def axes(ndim, kind, centeredh, nh):
    """the constructor's positional axes after taxis: 2-D (haxis, pxaxis), 3-D (hyaxis, hxaxis, pyaxis, pxaxis)"""
    def phys(pu, dh):
        return np.asarray(pu) / {"linear": dh / DT, "parabolic": dh * dh / DT, "hyperbolic": DT / dh}[kind]
    if ndim == 2:
        return haxis(nh, DH2, centeredh), phys(PU2[kind], DH2)
    (pyu, pxu), (dhy, dhx) = PU3[kind], DH3
    return (haxis(NH3[0], dhy, centeredh), haxis(NH3[1], dhx, centeredh), phys(pyu, dhy), phys(pxu, dhx))


def taxis(ndim):
    return np.arange(NT2 if ndim == 2 else NT3) * DT


def sizes(ndim, kind, nh):
    """(model values, data values) of one gather"""
    nt = NT2 if ndim == 2 else NT3
    if ndim == 2:
        return len(PU2[kind]) * nt, nh * nt
    return len(PU3[kind][0]) * len(PU3[kind][1]) * nt, NH3[0] * NH3[1] * nt


def case_inputs(ndim, kind, interp, centeredh, nh, dt):
    """global model x (NG gathers) and global data v, dtype dt"""
    nm, nd = sizes(ndim, kind, nh)
    rng = np.random.default_rng(900 + 97 * ndim + 13 * KINDS.index(kind) + 5 * int(interp) + 3 * int(centeredh)
                                + (nh or 0))
    x, xi = (rng.integers(-1, 2, NG * nm).astype(np.float64) for _ in range(2))
    v, vi = (rng.integers(-1, 2, NG * nd).astype(np.float64) for _ in range(2))
    if dt == "complex128":
        x, v = x + 1j * xi, v + 1j * vi
    return x.astype(dt), v.astype(dt)


def restated(ndim):
    """refshim's Radon2D / Radon3D class"""
    import importlib
    added = REFSHIM not in sys.path
    if added:
        sys.path.insert(0, REFSHIM)
    try:
        mod = importlib.import_module(f"pylops.signalprocessing.radon{ndim}d")
    finally:
        if added:
            sys.path.remove(REFSHIM)
    return getattr(mod, f"Radon{ndim}D")


def flow_axes():
    return np.arange(FLOW_NT) * DT, np.arange(FLOW_NH) * DH2, np.asarray(FLOW_PU) / (DH2 / DT)


def flow_inputs():
    """(sparse Radon models (FLOW_NG, npx, FLOW_NT), noisy gathers d (FLOW_NG * FLOW_NH * FLOW_NT,), alpha)"""
    t, h, p = flow_axes()
    R = restated(2)(t, h, p, kind="linear")
    rng = np.random.default_rng(52)
    m = np.zeros((FLOW_NG, p.size, FLOW_NT))
    for g in range(FLOW_NG):
        for _ in range(3):
            m[g, rng.integers(0, p.size), rng.integers(8, FLOW_NT - 8)] = rng.choice([-1.0, 1.0]) * (1 + rng.random())
    d = np.concatenate([R.matvec(mg.ravel()) for mg in m]) + 0.05 * rng.standard_normal(FLOW_NG * FLOW_NH * FLOW_NT)
    A = dense(R)
    alpha = 1.0 / float(np.abs(A).sum(0).max() * np.abs(A).sum(1).max())
    return m, d, alpha


def dense(op):
    return np.stack([op.matvec(e) for e in np.eye(op.shape[1])], 1)


def main():
    from make_golden import load_reference          # puts refshim/ (mpi4py, pylops) on the path
    from mpi4py import MPI
    pkg, mods = load_reference()
    DA = pkg.DistributedArray
    BD = mods["BlockDiag"].MPIBlockDiag
    FISTA = mods["cls_sparsity"].FISTA
    out = {}

    def t_op(rank, P, ndim, kind, interp, centeredh, nh, dt):
        x, v = case_inputs(ndim, kind, interp, centeredh, nh, dt)
        nm, nd = sizes(ndim, kind, nh)
        ny = rows_of(P, NG)
        R = restated(ndim)
        ops = [R(taxis(ndim), *axes(ndim, kind, centeredh, nh), kind=kind, centeredh=centeredh, interp=interp,
                 dtype="float32" if dt == "float32" else "float64") for _ in range(ny[rank])]
        Op = BD(ops, dtype=dt)
        return {"y": (Op @ DA.to_dist(x, local_shapes=[(r * nm,) for r in ny])).asarray(),
                "ya": (Op.H @ DA.to_dist(v, local_shapes=[(r * nd,) for r in ny])).asarray()}

    for c in cases():
        k = key(*c)
        ex = exact(c[1], c[2])
        runs = {}
        for dt in DTYPES:
            if dt == "complex128" and not complex_case(*c[1:4]):
                continue
            for P in (1, 2, 3):
                res = MPI.run_world(P, t_op, P, *c, dt)[0]
                if P == 1:
                    runs[dt] = res
                for n in ("y", "ya"):                      # each gather is computed alike: no dependence on P
                    assert np.array_equal(res[n], runs[dt][n])
        for n in ("y", "ya"):
            if ex:
                assert np.array_equal(runs["float32"][n], runs["float64"][n])
                out[f"{k}/{n}"] = encode(runs["float64"][n], ENC, np.int32)
            else:
                assert np.array_equal(runs["float32"][n], runs["float64"][n].astype(np.float32))
                out[f"{k}/{n}"] = runs["float64"][n]
            if "complex128" in runs:
                assert np.array_equal(runs["complex128"][n].real, runs["float64"][n])
                out[f"{k}/{n}i"] = encode(runs["complex128"][n].imag, ENC, np.int32)

    # flow, in float64
    t, h, p = flow_axes()
    R2 = restated(2)
    m, d, alpha = flow_inputs()
    out["flow/m"], out["flow/d"], out["flow/alpha"] = m.ravel(), d, np.asarray(alpha)
    out["flow/cond"] = np.asarray(np.linalg.cond(dense(R2(t, h, p, kind="linear"))))
    nd, nm = FLOW_NH * FLOW_NT, p.size * FLOW_NT

    def make_op(seed=None):
        if seed is None:
            return R2(t, h, p, kind="linear")

        class Jittered(R2):
            """the restated operator with every output scaled by 1 + 4 u g, g standard normal, seeded"""
            rng = np.random.default_rng(seed)

            def _matvec(self, x):
                y = super()._matvec(x)
                return y * (1 + 4 * 2.0 ** -53 * self.rng.standard_normal(y.shape))

            def _rmatvec(self, x):
                y = super()._rmatvec(x)
                return y * (1 + 4 * 2.0 ** -53 * self.rng.standard_normal(y.shape))
        return Jittered(t, h, p, kind="linear")

    def t_flow(rank, P, seed=None):
        ny = rows_of(P, FLOW_NG)
        Op = BD([make_op(seed) for _ in range(ny[rank])])
        dd = DA.to_dist(d, local_shapes=[(r * nd,) for r in ny])
        x0 = DA(global_shape=FLOW_NG * nm, local_shapes=[(r * nm,) for r in ny])
        x0[:] = 0
        x, iiter, cost = FISTA(Op).solve(dd, x0, niter=FLOW_NITER, eps=FLOW_EPS, alpha=alpha, tol=1e-10)
        return {"x": x.asarray(), "iiter": iiter, "cost": np.asarray(cost)}

    for P in (1, 2, 3):
        res = MPI.run_world(P, t_flow, P)[0]
        for k in ("x", "iiter", "cost"):
            out[f"flow/P{P}/{k}"] = np.asarray(res[k])
    spread = np.zeros(2)
    x1, c1 = out["flow/P1/x"], out["flow/P1/cost"]
    for seed in FLOW_JITTER_SEEDS:
        res = MPI.run_world(1, t_flow, 1, seed)[0]
        spread = np.maximum(spread, [np.abs(res["x"] - x1).max() / np.abs(x1).max(),
                                     (np.abs(res["cost"] - c1) / c1).max()])
    out["flow/spread"] = spread
    print(f"flow: cond {float(out['flow/cond']):.3e}, spread {spread}, cost {c1[0]:.3e} -> {c1[-1]:.3e}, "
          f"alpha {alpha:.3e}")

    path = os.path.join(HERE, os.environ.get("GOLDEN_OUT", "radon_golden.npz"))
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1e3:.0f} KB")


if __name__ == "__main__":
    main()
