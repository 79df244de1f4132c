"""Generate the Patch2D / Patch3D / Sliding1D fixtures by running the REAL reference's MPIBlockDiag and FISTA (a
pylops-mpi checkout named by PYLOPS_MPI_REFERENCE, imported unmodified through make_golden.load_reference) over
refshim's restated ``pylops.signalprocessing.Patch2D`` / ``Patch3D`` / ``Sliding1D`` (refshim/pylops/signalprocessing/
patch2d.py, patch3d.py, sliding1d.py) around the restated Radon2D / Radon3D and MatrixMult.

    PYLOPS_MPI_REFERENCE=<checkout> python tests/golden/make_golden_patch.py   # writes patch_golden.npz

NG sections split over P in {1, 2, 3} ranks, as make_golden_sliding.py does: rank r holds MPIBlockDiag([op for each
of its sections], dtype), float32 / float64 inner operators (float64 for complex data).  The Radon axes are
make_golden_radon's dyadic ones on a patch's traces and samples, MatrixMult's entries and all inputs are in
{-1, 0, 1}, and a hanning taper with nover = 3 on every tapered axis is {0, 1/2, 1} per axis, so its products are
dyadic: the outputs of those cases (``exact``) are the SAME in float64, float32 and complex128 and at every P (all
checked here), stored once, losslessly, as int32 of ENC * y.  Cosine tapers and hyperbolic curves with interpolation
are not dyadic: those outputs are stored as the float64 run.

  op/{geom}/{inner}[/{kind}/i{interp}]/{y,ya}     gathered forward of x / adjoint of v;  .../{yi,yai} imaginary parts

Flow: local time-space linear-Radon denoising.  FLOW_NG sections of FLOW_N traces and FLOW_NT samples, each a few
hyperbolic (curved) events plus seeded noise; then FISTA on MPIBlockDiag([Patch2D(Radon2D(linear))]), x0 = 0,
FLOW_NITER iterations, sparsity FLOW_EPS, alpha = 1 / (||A||_1 ||A||_inf) of one section's dense matrix.  ``cond`` and
``spread`` (4-ulp jitter of every apply, over FLOW_JITTER_SEEDS at P = 1) as in make_golden_sliding.

  flow/d, flow/alpha, flow/cond, flow/spread, flow/P{P}/{x,iiter,cost}
"""
import importlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REFSHIM = os.path.join(HERE, "refshim")
sys.path.insert(0, HERE)
import make_golden_radon as mgr  # noqa: E402
from fixture_codec import encode, rows_of  # noqa: E402

NG = 3
ENC = 1024       # stored value = ENC * y, exact in int32
DTYPES = ("float64", "float32", "complex128")
KINDS = mgr.KINDS

# geometry: (ndim, dimsd, nwin, nover, tapertype); ndim 1 is Sliding1D, 2 Patch2D, 3 Patch3D
GEOMS = {
    "hann2": (2, (22, 20), (8, 8), (3, 3), "hanning"),     # 3 x 3 patches, traces 18 .. 21 and samples 18, 19 past
    "single2": (2, (8, 20), (8, 8), (3, 3), "hanning"),   # one patch along the traces
    "nover0": (2, (16, 20), (8, 8), (0, 3), "hanning"),   # nover = 0 along the traces
    "cos2": (2, (22, 20), (10, 8), (4, 3), "cosine"),
    "hann3": (3, (9, 10, 14), (6, 6, 8), (3, 3, 3), "hanning"),   # 2 x 2 x 2, trace column 9 and sample 13 past
    "single3": (3, (6, 10, 16), (6, 6, 8), (3, 3, 0), "hanning"),  # one patch along y, nover = 0 along t
    "cos3": (3, (9, 9, 14), (6, 6, 8), (3, 3, 3), "cosine"),
    "hann1": (1, 22, 8, 3, "hanning"),
    "cos1": (1, 21, 10, 4, "cosine"),
}
CLASS = {1: "Sliding1D", 2: "Patch2D", 3: "Patch3D"}
NOP_MM = {1: (3,), 2: (2, 2), 3: (1, 1, 3)}      # MatrixMult's model per window

FLOW_NG, FLOW_N, FLOW_NT, FLOW_NITER, FLOW_EPS = 3, 24, 64, 30, 0.1
FLOW_NWIN, FLOW_NOVER = (12, 32), (6, 16)
FLOW_PU = tuple(np.arange(-2.0, 2.01, 0.25))
FLOW_JITTER_SEEDS = (1, 2, 3)


def cases():
    """(inner, kind, interp, geom): every Radon kind x interp on the hanning geometries, linear with interpolation on
    the others, hyperbolic with interpolation on the cosine ones, MatrixMult for each class"""
    out = []
    for g in ("hann2", "hann3"):
        for kind in KINDS:
            for interp in (True, False):
                out.append(("radon", kind, interp, g))
    for g in ("single2", "nover0", "cos2", "single3", "cos3"):
        out.append(("radon", "linear", True, g))
    out += [("radon", "hyperbolic", True, "cos2"), ("radon", "hyperbolic", True, "cos3")]
    out += [("matrix", None, None, g) for g in ("hann2", "nover0", "hann3", "hann1", "cos1")]
    return out


def key(inner, kind, interp, geom):
    return f"op/{geom}/{inner}" + ("" if kind is None else f"/{kind}/i{int(interp)}")


def exact(inner, kind, interp, geom):
    return GEOMS[geom][4] != "cosine" and (inner == "matrix" or mgr.exact(kind, interp))


def restated(name):
    """refshim's class ``name`` of pylops.signalprocessing.{patch2d, patch3d, sliding1d}, or pylops.MatrixMult"""
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


def _phys(kind, pu, d):
    return np.asarray(pu) / {"linear": d / mgr.DT, "parabolic": d * d / mgr.DT, "hyperbolic": mgr.DT / d}[kind]


def inner_spec(inner, kind, interp, geom):
    """(constructor, args, kwargs, nop) of the window operator: ``constructor(*args, **kwargs, dtype=...)``"""
    ndim, _, nwin, _, _ = GEOMS[geom]
    if inner == "matrix":
        nop = NOP_MM[ndim]
        nd = int(np.prod(nwin))
        A = np.random.default_rng(170 + 3 * ndim + len(geom)).integers(-1, 2, (nd, int(np.prod(nop)))).astype(float)
        return "MatrixMult", (A,), {}, nop
    t = np.arange(nwin[-1]) * mgr.DT
    if ndim == 2:
        args = (t, mgr.haxis(nwin[0], mgr.DH2, True), _phys(kind, mgr.PU2[kind], mgr.DH2))
        nop = (len(mgr.PU2[kind]), nwin[1])
    else:
        (pyu, pxu), (dhy, dhx) = mgr.PU3[kind], mgr.DH3
        args = (t, mgr.haxis(nwin[0], dhy, True), mgr.haxis(nwin[1], dhx, True), _phys(kind, pyu, dhy),
                _phys(kind, pxu, dhx))
        nop = (len(pyu), len(pxu), nwin[2])
    return f"Radon{ndim}D", args, {"kind": kind, "centeredh": True, "interp": interp}, nop


def outer_spec(c):
    """(class name, dims, dimsd, nwin, nover, extra kwargs, tapertype) of one section's operator"""
    ndim, dimsd, nwin, nover, tap = GEOMS[c[3]]
    nop = inner_spec(*c)[3]
    if ndim == 1:
        nwins = len(np.arange(0, dimsd - nwin + 1, nwin - nover))
        return "Sliding1D", nwins * nop[0], dimsd, nwin, nover, {}, tap
    nwins = [len(np.arange(0, dimsd[a] - nwin[a] + 1, nwin[a] - nover[a])) for a in range(ndim)]
    dims = tuple(w * n for w, n in zip(nwins, nop))
    return CLASS[ndim], dims, dimsd, nwin, nover, {"nop": nop}, tap


def sizes(c):
    _, dims, dimsd = outer_spec(c)[:3]
    return int(np.prod(dims)), int(np.prod(dimsd))


def make(c, dt, lib):
    """one section's operator, from ``lib``: a callable giving the inner classes and the window classes by name"""
    cname, args, kw, _ = inner_spec(*c)
    odt = "float32" if dt == "float32" else "float64"
    if cname == "MatrixMult":
        args = (args[0].astype(odt),)
    Op = lib(cname)(*args, **kw, dtype=odt)
    sname, dims, dimsd, nwin, nover, extra, tap = outer_spec(c)
    return lib(sname)(Op, dims, dimsd, nwin, nover, tapertype=tap, **extra)


def case_inputs(c, dt):
    """global model x (NG sections) and global data v, dtype dt"""
    nm, nd = sizes(c)
    rng = np.random.default_rng(2300 + sum(map(ord, key(*c))))
    x, xi = (rng.integers(-1, 2, NG * nm).astype(np.float64) for _ in range(2))
    v, vi = (rng.integers(-1, 2, NG * nd).astype(np.float64) for _ in range(2))
    if dt == "complex128":
        x, v = x + 1j * xi, v + 1j * vi
    return x.astype(dt), v.astype(dt)


def refshim_lib(name):
    return mgr.restated(2) if name == "Radon2D" else mgr.restated(3) if name == "Radon3D" else restated(name)


def flow_ops(lib):
    t = np.arange(FLOW_NWIN[1]) * mgr.DT
    h, p = np.arange(FLOW_NWIN[0]) * mgr.DH2, np.asarray(FLOW_PU) / (mgr.DH2 / mgr.DT)
    R = lib("Radon2D")(t, h, p, kind="linear")
    nop = (p.size, FLOW_NWIN[1])
    nwins = [len(np.arange(0, n - w + 1, w - o)) for n, w, o in zip((FLOW_N, FLOW_NT), FLOW_NWIN, FLOW_NOVER)]
    dims = (nwins[0] * nop[0], nwins[1] * nop[1])
    return lib("Patch2D")(R, dims, (FLOW_N, FLOW_NT), FLOW_NWIN, FLOW_NOVER, nop)


def flow_dense(P):
    """one section's dense matrix, from the restated Radon's dense matrix and the patches' tapers"""
    M = mgr.dense(P.Op)
    out = np.zeros(P.shape)
    nm = M.shape[1]
    cols = np.arange(FLOW_NWIN[0])[:, None] * FLOW_NT + np.arange(FLOW_NWIN[1])[None, :]
    for i0, a in enumerate(P.starts[0]):
        for i1, b in enumerate(P.starts[1]):
            w = i0 * len(P.starts[1]) + i1
            rows = (a * FLOW_NT + b + cols).ravel()
            out[rows, w * nm:(w + 1) * nm] += P.taps[w].astype(np.float64).ravel()[:, None] * M
    return out


def flow_inputs():
    """(noisy sections d (FLOW_NG * FLOW_N * FLOW_NT,), alpha)"""
    P = flow_ops(refshim_lib)
    rng = np.random.default_rng(71)
    d = np.zeros((FLOW_NG, FLOW_N, FLOW_NT))
    x = np.arange(FLOW_N) - FLOW_N / 2
    for g in range(FLOW_NG):
        for _ in range(3):            # hyperbolic events: locally linear in a patch, curved over the section
            t0, v = rng.uniform(8, FLOW_NT - 24), rng.uniform(0.6, 1.5)
            it = np.rint(np.sqrt(t0 * t0 + (x / v) ** 2)).astype(int)
            ok = it < FLOW_NT
            d[g, np.arange(FLOW_N)[ok], it[ok]] += rng.choice([-1.0, 1.0]) * (1 + rng.random())
    d = d.ravel() + 0.05 * rng.standard_normal(d.size)
    A = flow_dense(P)
    alpha = 1.0 / float(np.abs(A).sum(0).max() * np.abs(A).sum(1).max())
    return d, alpha


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
                assert np.array_equal(runs["float32"][n], runs["float64"][n]), (k, n)
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
        P2 = restated("Patch2D")

        class Jittered(P2):
            """the restated operator with every output scaled by 1 + 4 u g, g standard normal, seeded"""
            rng = np.random.default_rng(seed)

            def _matvec(self, x):
                y = super()._matvec(x)
                return y * (1 + 4 * 2.0 ** -53 * self.rng.standard_normal(y.shape))

            def _rmatvec(self, x):
                y = super()._rmatvec(x)
                return y * (1 + 4 * 2.0 ** -53 * self.rng.standard_normal(y.shape))
        return lambda name: Jittered if name == "Patch2D" else refshim_lib(name)

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

    path = os.path.join(HERE, os.environ.get("GOLDEN_OUT", "patch_golden.npz"))
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1e3:.0f} KB")


if __name__ == "__main__":
    main()
