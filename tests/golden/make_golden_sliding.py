"""Generate the Sliding2D / Sliding3D fixtures by running the REAL reference's MPIBlockDiag and FISTA (a pylops-mpi
checkout named by PYLOPS_MPI_REFERENCE, imported unmodified through make_golden.load_reference) over refshim's
restated ``pylops.signalprocessing.Sliding2D`` / ``Sliding3D`` (refshim/pylops/signalprocessing/sliding2d.py,
sliding3d.py) around the restated Radon2D / Radon3D and MatrixMult.

    PYLOPS_MPI_REFERENCE=<checkout> python tests/golden/make_golden_sliding.py   # writes sliding_golden.npz

NG sections split over P in {1, 2, 3} ranks: rank r holds MPIBlockDiag([Sliding(...) for each of its sections],
dtype), float32 / float64 inner operators (float64 for complex data) and dtype the data's.  The Radon axes are
make_golden_radon's dyadic ones, MatrixMult's entries and all inputs are in {-1, 0, 1}, and a hanning taper with
nover = 3 is {0, 1/2, 1}: the outputs of those cases (``exact``) are multiples of 1/128, the SAME in float64,
float32 and complex128 and at every P (all checked here), stored once, losslessly, as int32 of ENC * y.  Cosine
tapers with nover = 4 and hyperbolic curves with interpolation are not dyadic: those outputs are stored as the float64
run and the tests compare other dtypes under a rounding bound.

  op/{name}/{y,ya}       gathered forward of x / adjoint of v;  .../{yi,yai}  imaginary parts (exact cases)

Flow: local linear-Radon denoising.  FLOW_NG sections of FLOW_N traces and FLOW_NT samples, each a few locally
linear events plus seeded noise, split over the ranks; then FISTA on MPIBlockDiag([Sliding2D(Radon2D(linear))]),
x0 = 0, FLOW_NITER iterations, sparsity FLOW_EPS, alpha = 1 / (||A||_1 ||A||_inf) of one section's dense matrix.
``cond`` and ``spread`` (4-ulp jitter of every apply, over FLOW_JITTER_SEEDS at P = 1) as in make_golden_radon.

  flow/d, flow/alpha, flow/cond, flow/spread, flow/P{P}/{x,iiter,cost}
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REFSHIM = os.path.join(HERE, "refshim")
sys.path.insert(0, HERE)
import make_golden_radon as mgr  # noqa: E402
from fixture_codec import encode, rows_of  # noqa: E402

NG = 3
ENC = 256        # stored value = ENC * y, exact in int32
DTYPES = ("float64", "float32", "complex128")
KINDS = mgr.KINDS
NOP_MM = (3, 5)  # MatrixMult's model per window, 2-D; 3-D (2, 2, 3)

# geometry: (ndim, n (2-D) or (n0, n1), nwin, nover, tapertype)
GEOMS = {
    "hann": (2, 22, 8, 3, "hanning"),           # three windows, traces 18 .. 21 past the last one
    "none": (2, 18, 8, 3, None),
    "nover0": (2, 16, 8, 0, "hanning"),
    "single": (2, 8, 8, 3, "hanning"),          # nwin == n: one window
    "cosine": (2, 22, 10, 4, "cosine"),
    "hann3": (3, (9, 10), (6, 6), (3, 3), "hanning"),   # 2 x 2 windows, trace column 9 past the last one
    "single3": (3, (6, 10), (6, 6), (3, 3), None),      # one window along axis 0
    "cos3": (3, (9, 9), (6, 6), (3, 3), "cosine"),
}

FLOW_NG, FLOW_NT, FLOW_N, FLOW_NWIN, FLOW_NOVER, FLOW_NITER, FLOW_EPS = 3, 64, 24, 12, 6, 30, 0.1
FLOW_PU = tuple(np.arange(-2.0, 2.01, 0.25))
FLOW_JITTER_SEEDS = (1, 2, 3)


def cases():
    """(name, inner, kind, interp, geom): every Radon kind x interp on the hanning geometries, linear with
    interpolation on the others, hyperbolic with interpolation on the cosine ones, MatrixMult on each dimension"""
    out = []
    for g in ("hann", "hann3"):
        for kind in KINDS:
            for interp in (True, False):
                out.append(("radon", kind, interp, g))
    for g in ("none", "nover0", "single", "cosine", "single3", "cos3"):
        out.append(("radon", "linear", True, g))
    out += [("radon", "hyperbolic", True, "cosine"), ("radon", "hyperbolic", True, "cos3")]
    out += [("matrix", None, None, g) for g in ("hann", "nover0", "hann3", "cos3")]
    return out


def key(inner, kind, interp, geom):
    return f"op/{geom}/{inner}" + ("" if kind is None else f"/{kind}/i{int(interp)}")


def exact(inner, kind, interp, geom):
    return GEOMS[geom][4] != "cosine" and (inner == "matrix" or mgr.exact(kind, interp))


def restated(name):
    """refshim's class ``name`` of pylops.signalprocessing.{sliding2d, sliding3d}, or pylops.MatrixMult"""
    import importlib
    added = REFSHIM not in sys.path
    if added:
        sys.path.insert(0, REFSHIM)
    try:
        if name == "MatrixMult":
            return importlib.import_module("pylops").MatrixMult
        mod = importlib.import_module(f"pylops.signalprocessing.{name.lower()}")
    finally:
        if added:
            sys.path.remove(REFSHIM)
    return getattr(mod, name)


def inner_spec(inner, kind, interp, geom):
    """(constructor, args, kwargs, nop) of the window operator: ``constructor(*args, **kwargs, dtype=...)``"""
    ndim, n, nwin, nover, tap = GEOMS[geom]
    nt = mgr.NT2 if ndim == 2 else mgr.NT3
    if inner == "matrix":
        nop = NOP_MM if ndim == 2 else (2, 2, 3)
        nd = (nwin if ndim == 2 else nwin[0] * nwin[1]) * nt
        A = np.random.default_rng(70 + 3 * ndim + len(geom)).integers(-1, 2, (nd, int(np.prod(nop)))).astype(float)
        return "MatrixMult", (A,), {}, nop
    dh = mgr.DH2 if ndim == 2 else mgr.DH3

    def phys(pu, d):
        return np.asarray(pu) / {"linear": d / mgr.DT, "parabolic": d * d / mgr.DT, "hyperbolic": mgr.DT / d}[kind]
    t = np.arange(nt) * mgr.DT
    if ndim == 2:
        args = (t, mgr.haxis(nwin, dh, True), phys(mgr.PU2[kind], dh))
        nop = (len(mgr.PU2[kind]), nt)
    else:
        (pyu, pxu), (dhy, dhx) = mgr.PU3[kind], dh
        args = (t, mgr.haxis(nwin[0], dhy, True), mgr.haxis(nwin[1], dhx, True), phys(pyu, dhy), phys(pxu, dhx))
        nop = (len(pyu), len(pxu), nt)
    return f"Radon{ndim}D", args, {"kind": kind, "centeredh": True, "interp": interp}, nop


def sliding_spec(inner, kind, interp, geom):
    """(Sliding class name, dims, dimsd, nwin, nover, extra kwargs, tapertype)"""
    ndim, n, nwin, nover, tap = GEOMS[geom]
    nt = mgr.NT2 if ndim == 2 else mgr.NT3
    nop = inner_spec(inner, kind, interp, geom)[3]
    if ndim == 2:
        nwins = len(np.arange(0, n - nwin + 1, nwin - nover))
        return "Sliding2D", (nwins * nop[0], nop[1]), (n, nt), nwin, nover, {}, tap
    nw = [len(np.arange(0, n[a] - nwin[a] + 1, nwin[a] - nover[a])) for a in (0, 1)]
    return "Sliding3D", (nw[0] * nop[0], nw[1] * nop[1], nop[2]), (n[0], n[1], nt), nwin, nover, {"nop": nop}, tap


def sizes(c):
    _, dims, dimsd = sliding_spec(*c)[:3]
    return int(np.prod(dims)), int(np.prod(dimsd))


def make(c, dt, lib):
    """one section's operator, from ``lib``: a module-like object with the inner classes and Sliding2D / 3D"""
    cname, args, kw, _ = inner_spec(*c)
    odt = "float32" if dt == "float32" else "float64"
    if cname == "MatrixMult":
        args = (args[0].astype(odt),)
    Op = lib(cname)(*args, **kw, dtype=odt)
    sname, dims, dimsd, nwin, nover, extra, tap = sliding_spec(*c)
    return lib(sname)(Op, dims, dimsd, nwin, nover, tapertype=tap, **extra)


def case_inputs(c, dt):
    """global model x (NG sections) and global data v, dtype dt"""
    nm, nd = sizes(c)
    rng = np.random.default_rng(1300 + sum(map(ord, key(*c))))
    x, xi = (rng.integers(-1, 2, NG * nm).astype(np.float64) for _ in range(2))
    v, vi = (rng.integers(-1, 2, NG * nd).astype(np.float64) for _ in range(2))
    if dt == "complex128":
        x, v = x + 1j * xi, v + 1j * vi
    return x.astype(dt), v.astype(dt)


def flow_ops(lib, seed=None):
    t, h, p = np.arange(FLOW_NT) * mgr.DT, np.arange(FLOW_NWIN) * mgr.DH2, np.asarray(FLOW_PU) / (mgr.DH2 / mgr.DT)
    R = lib("Radon2D")(t, h, p, kind="linear")
    nwins = len(np.arange(0, FLOW_N - FLOW_NWIN + 1, FLOW_NWIN - FLOW_NOVER))
    return lib("Sliding2D")(R, (nwins * p.size, FLOW_NT), (FLOW_N, FLOW_NT), FLOW_NWIN, FLOW_NOVER)


def refshim_lib(name):
    return mgr.restated(2) if name == "Radon2D" else mgr.restated(3) if name == "Radon3D" else restated(name)


def flow_inputs():
    """(noisy sections d (FLOW_NG * FLOW_N * FLOW_NT,), alpha)"""
    S = flow_ops(refshim_lib)
    rng = np.random.default_rng(61)
    d = np.zeros((FLOW_NG, FLOW_N, FLOW_NT))
    tr = np.arange(FLOW_N)
    for g in range(FLOW_NG):
        for _ in range(3):            # events whose slope changes halfway across the section
            t0, s1, s2 = rng.integers(10, FLOW_NT - 20), rng.uniform(-0.8, 0.8), rng.uniform(-0.8, 0.8)
            tt = t0 + np.where(tr < FLOW_N // 2, s1 * tr, s1 * (FLOW_N // 2) + s2 * (tr - FLOW_N // 2))
            it = np.rint(tt).astype(int)
            ok = (it >= 0) & (it < FLOW_NT)
            d[g, tr[ok], it[ok]] += rng.choice([-1.0, 1.0]) * (1 + rng.random())
    d = d.ravel() + 0.05 * rng.standard_normal(d.size)
    A = flow_dense(S)
    alpha = 1.0 / float(np.abs(A).sum(0).max() * np.abs(A).sum(1).max())
    return d, alpha


def flow_dense(S):
    """one section's dense matrix, from the restated Radon's dense matrix and the windows' tapers"""
    R = S.Op
    M = mgr.dense(R)
    out = np.zeros(S.shape)
    nm, nt = R.shape[1], FLOW_NT
    for w, s in enumerate(S.starts[1]):
        tap = S.taps[w][0].astype(np.float64).ravel()
        out[s * nt:(s + FLOW_NWIN) * nt, w * nm:(w + 1) * nm] += tap[:, None] * M
    return out


def main():
    from make_golden import load_reference          # puts refshim/ (mpi4py, pylops) on the path
    from mpi4py import MPI
    pkg, mods = load_reference()
    DA = pkg.DistributedArray
    BD = mods["BlockDiag"].MPIBlockDiag
    FISTA = mods["cls_sparsity"].FISTA
    out = {}

    def t_op(rank, P, c, dt):
        x, v = case_inputs(c, dt)
        nm, nd = sizes(c)
        ny = rows_of(P, NG)
        Op = BD([make(c, dt, refshim_lib) for _ in range(ny[rank])], dtype=dt)
        return {"y": (Op @ DA.to_dist(x, local_shapes=[(r * nm,) for r in ny])).asarray(),
                "ya": (Op.H @ DA.to_dist(v, local_shapes=[(r * nd,) for r in ny])).asarray()}

    for c in cases():
        k = key(*c)
        ex = exact(*c)
        runs = {}
        for dt in DTYPES:
            if dt == "complex128" and not ex:
                continue
            for P in (1, 2, 3):
                res = MPI.run_world(P, t_op, P, c, dt)[0]
                if P == 1:
                    runs[dt] = res
                for n in ("y", "ya"):
                    assert np.array_equal(res[n], runs[dt][n])
        for n in ("y", "ya"):
            assert np.count_nonzero(runs["float64"][n]) > 0, (k, n)
            if ex:
                assert np.array_equal(runs["float32"][n], runs["float64"][n])
                assert np.array_equal(runs["complex128"][n].real, runs["float64"][n])
                out[f"{k}/{n}"] = encode(runs["float64"][n], ENC, np.int32)
                out[f"{k}/{n}i"] = encode(runs["complex128"][n].imag, ENC, np.int32)
            else:
                out[f"{k}/{n}"] = runs["float64"][n]

    # flow, in float64
    d, alpha = flow_inputs()
    out["flow/d"], out["flow/alpha"] = d, np.asarray(alpha)
    out["flow/cond"] = np.asarray(np.linalg.cond(flow_dense(flow_ops(refshim_lib))))
    nd = FLOW_N * FLOW_NT
    nm = flow_ops(refshim_lib).shape[1]

    def jittered(seed):
        S2 = restated("Sliding2D")

        class Jittered(S2):
            """the restated operator with every output scaled by 1 + 4 u g, g standard normal, seeded"""
            rng = np.random.default_rng(seed)

            def _matvec(self, x):
                y = super()._matvec(x)
                return y * (1 + 4 * 2.0 ** -53 * self.rng.standard_normal(y.shape))

            def _rmatvec(self, x):
                y = super()._rmatvec(x)
                return y * (1 + 4 * 2.0 ** -53 * self.rng.standard_normal(y.shape))
        return lambda name: Jittered if name == "Sliding2D" else refshim_lib(name)

    def t_flow(rank, P, seed=None):
        ny = rows_of(P, FLOW_NG)
        lib = refshim_lib if seed is None else jittered(seed)
        Op = BD([flow_ops(lib) for _ in range(ny[rank])])
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

    path = os.path.join(HERE, os.environ.get("GOLDEN_OUT", "sliding_golden.npz"))
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1e3:.0f} KB")


if __name__ == "__main__":
    main()
