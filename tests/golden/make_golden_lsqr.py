"""Generate the LSQR fixtures by running scipy.sparse.linalg.lsqr (the definition LSQR follows) on the CPU.

    python tests/golden/make_golden_lsqr.py            # writes tests/golden/lsqr_golden.npz (byte-identical reruns)

Every parameter is passed explicitly (scipy's own defaults differ: atol = btol = 1e-6, calc_var=False).  For each case
``<name>/`` holds the inputs (``A`` dense, ``b``, ``x0``) and scipy's outputs: ``x istop itn r1norm r2norm anorm acond
arnorm xnorm var`` and ``cost``, the r1norm history, recorded by rerunning scipy with iter_lim = 1..itn (its iterations
are deterministic), and ``spread``: LSQR amplifies rounding as it converges, so eps does not bound how far the
device's iterates may lie from scipy's.  ``spread`` measures it on scipy's own loop (``transcription``, which is
scipy's loop bit for bit): both vector combinations of every iteration jittered by 4 ulps of the data's type per
component, three seeds, and for float32 data also scipy run in float32.  It holds the largest change of (x, var,
r1norm, r2norm, anorm, acond, arnorm, xnorm, cost history), each on the scale it is resolved to (``spread_of``).
float32 cases run scipy on the float64 values of the float32 data.

Dense cases (the tests apply ``A`` as an MPIBlockDiag of MatrixMult blocks, ``NBLK`` row/column blocks):
  consistent (istop 1), inconsistent (istop 2), illcond with conlim = 50 (istop 3), limit (istop 7), damped,
  x0 (non-zero x0), novar (calc_var=False), complex (complex128), float32.
Flow: tutorials/lsm.py's geometry through refshim's analytic Kirchhoff, all FLOW_NS sources stacked (``flow/``,
FLOW_NITER iterations) and one rank's sources of two (``lsm/``: what LSM.solve inverts).  The data are recomputed by
the tests; ``spread`` is the largest change of the image, relative to its largest entry, under the same jitter.

At no iteration of any case may a stopping test lie within 1e-6 (relative) of its threshold (all seven, the
``1 + t <= 1`` tests included), else rounding-order differences could move istop or itn: checked here with the scalar recurrence of
pylops_mpi_b200/optimization/lsqr_host.py, which reproduces scipy's loop bit for bit given scipy's reductions.
"""
import functools
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)

NBLK = 2
ATOL = BTOL = 1e-8
CONLIM = 1e8
FLOW_NITER = 100


@functools.lru_cache(maxsize=None)
def lsqr_host():
    """pylops_mpi_b200/optimization/lsqr_host.py without importing the package (which needs the CUDA library)"""
    spec = importlib.util.spec_from_file_location(
        "_lsqr_host", os.path.join(ROOT, "pylops_mpi_b200", "optimization", "lsqr_host.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _nsq(a):
    """np.linalg.norm(a) ** 2 before the square root, as NumPy sums it"""
    return float(a.real.dot(a.real) + a.imag.dot(a.imag)) if np.iscomplexobj(a) else float(a.dot(a))


def _jitter(a, rng, eps):
    """a with every real component moved by up to 4 units of eps (relative): a rounding that differs per element"""
    if rng is None:
        return a
    f = lambda: 1 + rng.integers(-4, 5, a.size) * eps                    # noqa: E731
    return a.real * f() + 1j * (a.imag * f()) if np.iscomplexobj(a) else a * f()


def transcription(A, b, damp, atol, btol, conlim, niter, calc_var, x0, rng=None, eps=0.0):
    """scipy's lsqr with its vectors and reductions, the scalars through lsqr_host: (scipy's outputs, per-iteration
    (test1, rtol, test2, test3, r1norm, tt1) at the finishing of each iteration).  With ``rng``, both vector
    combinations of every iteration are jittered by up to 4 eps per component (``_jitter``)."""
    H = lsqr_host()
    mv = A.matvec if hasattr(A, "matvec") else (lambda v: A @ v)
    rmv = A.rmatvec if hasattr(A, "rmatvec") else (lambda u: A.conj().T @ u)
    n = A.shape[1]
    x = np.zeros(n) if x0 is None else np.asarray(x0).copy()
    u = b if x0 is None else b - mv(x)
    bnorm = np.linalg.norm(b)
    beta = bnorm if x0 is None else np.linalg.norm(u)
    var = np.zeros(n)
    if beta > 0:
        u = (1 / beta) * u
        v = rmv(u)
        alfa = np.linalg.norm(v)
    else:
        v, alfa = x.copy(), 0
    if alfa > 0:
        v = (1 / alfa) * v
    w = v.copy()
    s = np.zeros(H._NSTATE)
    s[[H._ALFA, H._BETA, H._RHOBAR, H._PHIBAR, H._CS2, H._INV_ALFA]] = alfa, beta, alfa, beta, -1, \
        (1 / alfa if alfa > 0 else 1)
    s[[H._DAMP, H._DAMPSQ, H._ATOL, H._BTOL, H._CTOL, H._BNORM, H._ITER_LIM]] = damp, damp ** 2, atol, btol, \
        (1 / conlim if conlim > 0 else 0), bnorm, niter
    rows, tests = [], []
    for _ in range(niter):
        up = _jitter(mv(v) - alfa * u, rng, eps)
        s[H._BB] = _nsq(up)
        H.lsqr_scalars_host(s, 0)
        beta = s[H._BETA]
        if beta > 0:
            u = (1 / beta) * up
            vp = _jitter(rmv(u) - beta * v, rng, eps)
            s[H._AA] = _nsq(vp)
        else:
            u = up
        H.lsqr_scalars_host(s, 1)
        if beta > 0:
            alfa = s[H._ALFA]
            v = (1 / alfa) * vp if alfa > 0 else vp
        dk = s[H._INV_RHO] * w
        x = x + s[H._T1] * w
        w = v + s[H._T2] * w
        s[H._DD] = np.linalg.norm(dk) ** 2
        if calc_var:
            var = var + dk ** 2
        row = H.lsqr_scalars_host(s, 2)
        rows.append(row)
        tests.append((row[6], s[H._RTOL], row[7], 1 / (row[3] + H._EPS), row[0], s[H._TT1]))
        if row[8]:
            break
    r = rows[-1]
    return (x, int(r[8]), len(rows), r[0], r[1], r[2], r[3], r[4], r[5], var), tests


def check_margin(tests, atol, conlim):
    """at every iteration, no stopping test within 1e-6 (relative) of its threshold: test1 <= rtol, test2 <= atol,
    test3 <= ctol, and 1 + t <= 1 (t <= 2^-53) for t = test3, test2, tt1 (istop 6, 5, 4)"""
    ctol = 1 / conlim
    for it, (test1, rtol, test2, test3, _, tt1) in enumerate(tests):
        for val, thr in ((test1, rtol), (test2, atol), (test3, ctol), (test3, 2.0 ** -53), (test2, 2.0 ** -53),
                         (tt1, 2.0 ** -53)):
            assert abs(val - thr) > 1e-6 * thr, (it + 1, val, thr)


def spread_of(res, cost, rp, hist):
    """relative changes of a rerun, each on a scale the quantity is resolved to: x and var to their largest entry,
    r1norm, r2norm and the cost history to the initial residual norm cost[0], arnorm = |A^H r| to anorm * cost[0],
    anorm, acond and xnorm to themselves"""
    c0 = abs(cost[0])
    scale = [np.abs(res[0]).max(), max(np.abs(res[9]).max(), 1e-300), c0, c0, abs(res[5]), abs(res[6]),
             abs(res[5]) * c0, abs(res[8])]
    got = [np.abs(rp[0] - res[0]).max(), np.abs(rp[9] - res[9]).max()] + [abs(rp[k] - res[k]) for k in range(3, 9)]
    return [g / sc if sc else 0.0 for g, sc in zip(got, scale)] + \
        [float(np.max(np.abs(np.asarray(hist) - cost))) / c0]


def run_case(out, name, A, b, damp=0.0, atol=ATOL, btol=BTOL, conlim=CONLIM, niter=60, calc_var=True, x0=None,
             expect=None):
    from scipy.sparse.linalg import lsqr
    Aop = A.astype(np.complex128 if np.iscomplexobj(A) else np.float64)
    bb = b.astype(Aop.dtype)
    x00 = None if x0 is None else x0.astype(Aop.dtype)
    res = lsqr(Aop, bb, damp=damp, atol=atol, btol=btol, conlim=conlim, iter_lim=niter, calc_var=calc_var, x0=x00)
    tx, tests = transcription(Aop, bb, damp, atol, btol, conlim, niter, calc_var, x00)
    for a, c in zip(tx, res):
        np.testing.assert_array_equal(np.asarray(a), np.asarray(c))
    istop, itn = res[1], res[2]
    assert expect is None or istop == expect, (name, istop, expect)
    check_margin(tests, atol, conlim)
    cost = [np.linalg.norm(bb if x00 is None else bb - Aop @ x00)]
    cost += [lsqr(Aop, bb, damp=damp, atol=atol, btol=btol, conlim=conlim, iter_lim=k, calc_var=calc_var,
                  x0=x00)[3] for k in range(1, itn + 1)]
    assert cost[-1] == res[3] and np.array_equal(cost[1:], [t[4] for t in tests])
    # LSQR amplifies rounding as it converges, so eps does not bound the device's difference from scipy.  The spread
    # measures it: scipy's loop with both vector combinations of every iteration jittered by 4 ulps of the data's
    # type per component (the device rounds each of them differently), three seeds; for float32 data also scipy
    # run in float32 (its vectors stay float32)
    spread = np.zeros(9)
    eps = float(np.finfo(A.real.dtype).eps)
    for seed in range(3):
        rp, tp = transcription(Aop, bb, damp, atol, btol, conlim, niter, calc_var, x00,
                               rng=np.random.default_rng(seed), eps=eps)
        assert rp[1] == istop and rp[2] == itn, (name, rp[1], rp[2])
        spread = np.maximum(spread, spread_of(res, cost, rp, [cost[0]] + [t[4] for t in tp]))
    if A.dtype == np.float32:
        run32 = lambda k: lsqr(A, b, damp=damp, atol=atol, btol=btol, conlim=conlim, iter_lim=k,  # noqa: E731
                               calc_var=calc_var, x0=x0)
        rp = run32(niter)
        assert rp[1] == istop and rp[2] == itn
        spread = np.maximum(spread, spread_of(res, cost, rp, [np.linalg.norm(b if x0 is None else b - A @ x0)] +
                                              [run32(k)[3] for k in range(1, itn + 1)]))
    out[f"{name}/spread"] = spread
    out[f"{name}/A"], out[f"{name}/b"] = A, b
    out[f"{name}/x0"] = np.zeros(A.shape[1], A.dtype) if x0 is None else x0
    out[f"{name}/params"] = np.array([damp, atol, btol, conlim, niter, float(calc_var), float(x0 is not None)])
    for k, v in zip(("x", "istop", "itn", "r1norm", "r2norm", "anorm", "acond", "arnorm", "xnorm", "var"), res):
        out[f"{name}/{k}"] = np.asarray(v)
    out[f"{name}/cost"] = np.asarray(cost)


def blockdiag(blocks):
    m, n = sum(b.shape[0] for b in blocks), sum(b.shape[1] for b in blocks)
    A = np.zeros((m, n), blocks[0].dtype)
    i = j = 0
    for b in blocks:
        A[i:i + b.shape[0], j:j + b.shape[1]] = b
        i, j = i + b.shape[0], j + b.shape[1]
    return A


def dense_cases(out):
    rng = np.random.default_rng(2024)
    blk = lambda m, n: blockdiag([rng.standard_normal((m, n)) for _ in range(NBLK)])  # noqa: E731
    A = blk(40, 30) + 0.0
    run_case(out, "consistent", A, A @ rng.standard_normal(A.shape[1]), niter=200, expect=1)
    A = blk(40, 30)
    run_case(out, "inconsistent", A, rng.standard_normal(A.shape[0]), niter=200, expect=2)
    # ill-conditioned (singular values over two decades) with conlim = 50: the condition estimate stops it (istop 3)
    # at iteration 14, before rounding has grown (a 4-ulp jitter per iteration moves x by 4e-6 of its size; with six
    # decades and conlim = 1e3 the iterate at the stop moved by 25 %, pinning nothing but istop and itn)
    r7 = np.random.default_rng(7)
    U, _ = np.linalg.qr(r7.standard_normal((48, 48)))
    V, _ = np.linalg.qr(r7.standard_normal((32, 32)))
    S = np.zeros((48, 32))
    S[:32, :32] = np.diag(np.logspace(0, -2, 32))
    Ai = U @ S @ V.T
    run_case(out, "illcond", blockdiag([Ai, Ai[::-1]]), r7.standard_normal(96), conlim=50, niter=200, expect=3)
    A = blk(40, 30)
    run_case(out, "limit", A, rng.standard_normal(A.shape[0]), niter=12, expect=7)
    A = blk(40, 30)
    run_case(out, "damped", A, rng.standard_normal(A.shape[0]), damp=0.7, niter=40)
    A = blk(40, 30)
    run_case(out, "x0", A, rng.standard_normal(A.shape[0]), damp=0.2, x0=rng.standard_normal(A.shape[1]), niter=40)
    A = blk(40, 30)
    run_case(out, "novar", A, rng.standard_normal(A.shape[0]), calc_var=False, niter=40)
    A = blockdiag([rng.standard_normal((40, 30)) + 1j * rng.standard_normal((40, 30)) for _ in range(NBLK)])
    run_case(out, "complex", A, rng.standard_normal(80) + 1j * rng.standard_normal(80), damp=0.3,
             x0=rng.standard_normal(60) + 1j * rng.standard_normal(60), niter=40)
    A = blk(40, 30).astype(np.float32)
    run_case(out, "float32", A, rng.standard_normal(A.shape[0]).astype(np.float32), niter=25, expect=7)


def flow_cases(out):
    from scipy.sparse.linalg import LinearOperator, lsqr
    import make_golden_kirchhoff as mgk
    kirchhoff, _ = mgk.refshim()
    for name, P, rank in (("flow", 1, None), ("lsm", 2, 0)):
        z, x, t, srcs, recs, v0, wav, wavc, refl = mgk.flow_setup(P, rank)
        Op = kirchhoff.Kirchhoff(z, x, t, srcs, recs, v0, wav, wavc, mode="analytic")
        A = LinearOperator(Op.shape, matvec=Op.matvec, rmatvec=Op.rmatvec, dtype=np.float64)
        d = Op.matvec(refl.ravel())
        res = lsqr(A, d, damp=0.0, atol=ATOL, btol=BTOL, conlim=CONLIM, iter_lim=FLOW_NITER, calc_var=True)
        tx, tests = transcription(A, d, 0.0, ATOL, BTOL, CONLIM, FLOW_NITER, True, None)
        for a, c in zip(tx, res):
            np.testing.assert_array_equal(np.asarray(a), np.asarray(c))
        check_margin(tests, ATOL, CONLIM)
        spread = 0.0
        for seed in range(3):
            rp, _ = transcription(A, d, 0.0, ATOL, BTOL, CONLIM, FLOW_NITER, True, None,
                                  rng=np.random.default_rng(seed), eps=float(np.finfo(np.float64).eps))
            assert rp[1] == res[1] and rp[2] == res[2]
            spread = max(spread, float(np.abs(rp[0] - res[0]).max() / np.abs(res[0]).max()))
        for k, v in zip(("x", "istop", "itn", "r1norm", "r2norm", "anorm", "acond", "arnorm", "xnorm", "var"), res):
            out[f"{name}/{k}"] = np.asarray(v)
        out[f"{name}/spread"] = np.asarray(spread)
        out[f"{name}/geometry"] = np.array([P, -1 if rank is None else rank])


def main():
    out = {}
    dense_cases(out)
    flow_cases(out)
    path = os.path.join(HERE, os.environ.get("GOLDEN_OUT", "lsqr_golden.npz"))
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1e6:.3f} MB")


if __name__ == "__main__":
    main()
