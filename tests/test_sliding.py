"""Rank-local Sliding2D / Sliding3D (pylops.signalprocessing.Sliding2D / Sliding3D inside MPIBlockDiag): windows of
``nwin`` traces every ``nwin - nover`` traces along the section's trace axes, one inner operator per window, tapered
and overlap-added:

    y = sum over i0 ascending of (sum over i1 ascending of R_w^T (tap_w * Op x_w)),   x_w = Op^H (tap_w * R_w d)

CPU: refshim's restatement (tests/golden/refshim/pylops/signalprocessing/sliding2d.py, sliding3d.py,
utils/tapers.py) against a dense matrix built directly from that definition, argument errors, the library's host
tapers and design helpers, and the fixtures of tests/golden/sliding_golden.npz (made by make_golden_sliding.py: the
reference's MPIBlockDiag and FISTA over the restatement).  GPU: the b2_sliding and b2_radon_windows kernels through
the C ABI and the operators through the public interface."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_radon as mgr_radon  # noqa: E402
import make_golden_sliding as mgs  # noqa: E402
from fixture_codec import decode, rows_of  # noqa: E402
from op_checks import (assert_cgls_replay_matches_steps, assert_rejected, guarded_twice, host,  # noqa: E402
                       needs_gpus, run_on_ranks)

GOLD = np.load(os.path.join(HERE, "golden", "sliding_golden.npz"), allow_pickle=False)
CASES = mgs.cases()
U64, U32 = 2.0 ** -53, 2.0 ** -24


# ---------------------------------------------------------------------------------------------------------------
# the definition, built directly
# ---------------------------------------------------------------------------------------------------------------
def rise(ntap, tapertype):
    """the first ntap samples of a taper, from its formula (hanning: NumPy's, 0.5 + 0.5 cos(pi n / (M - 1)) for
    n = 1 - M, 3 - M, ... on M = 2 ntap - 1 samples)"""
    k = np.arange(ntap)
    if tapertype == "hanning":
        m = 2 * ntap - 1
        return 0.5 + 0.5 * np.cos(np.pi * (1 - m + 2 * k) / (m - 1)) if ntap > 1 else np.ones(ntap)
    if ntap <= 1:
        return np.ones(0)
    c = ntap - 1
    return (0.5 * (np.cos((k - c) * np.pi / c) + 1.0)) ** (2 if tapertype == "cosinesquare" else 1)


def axis_tapers(n, nwin, nover, tapertype):
    """(starts, (nwins, nwin) tapers): windows every nwin - nover traces, the first window's leading and the last
    window's trailing nover samples 1 (one window: the trailing ones only)"""
    starts = np.arange(0, n - nwin + 1, nwin - nover)
    tap = np.ones(nwin)
    if tapertype is not None:
        r = rise(nover, tapertype)
        tap[:len(r)] = r
        tap[nwin - len(r):] = r[::-1]
    taps = np.tile(tap, (len(starts), 1))
    if len(starts) > 1:
        taps[0, :nover] = 1
    taps[-1, nwin - nover:] = 1
    return starts, taps


def dense_sliding(A, n, nwin, nover, tapertype, inner):
    """the matrix of a sliding operator with windows on axes (0, 1) of an (n0, n1, inner) section (2-D: n0 = 1),
    window w = i0 * nw1 + i1 applying the dense window matrix A then its taper"""
    (s0, t0), (s1, t1) = (axis_tapers(n[a], nwin[a], nover[a], tapertype) for a in (0, 1))
    nw = len(s0) * len(s1)
    M = np.zeros((n[0] * n[1] * inner, nw * A.shape[1]))
    for i0, a in enumerate(s0):
        for i1, b in enumerate(s1):
            w = i0 * len(s1) + i1
            tap = np.outer(t0[i0], t1[i1])
            for j0 in range(nwin[0]):
                for j1 in range(nwin[1]):
                    rows = ((a + j0) * n[1] + b + j1) * inner + np.arange(inner)
                    arow = (j0 * nwin[1] + j1) * inner + np.arange(inner)
                    M[rows, w * A.shape[1]:(w + 1) * A.shape[1]] += tap[j0, j1] * A[arow]
    return M


def restated(name):
    return mgs.restated(name)


# (2-D: n, nwin, nover; 3-D: pairs), tapertype
DEFS = [((1, 22), (1, 8), (0, 3), "hanning"), ((1, 16), (1, 8), (0, 0), "hanning"), ((1, 8), (1, 8), (0, 3), "hanning"),
        ((1, 21), (1, 10), (0, 4), "cosine"), ((1, 20), (1, 9), (0, 2), "cosinesquare"), ((1, 19), (1, 6), (0, 2), None),
        ((9, 10), (6, 6), (3, 3), "hanning"), ((6, 11), (6, 5), (2, 2), "cosine"), ((9, 7), (4, 7), (2, 3), None)]


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", DEFS, ids=[f"{d[0]}-{d[1]}-{d[2]}-{d[3]}" for d in DEFS])
def test_restatement_is_the_dense_definition(geom):
    n, nwin, nover, tapertype = geom
    rng = np.random.default_rng(sum(n) + sum(nwin))
    inner = 3
    nop = 4
    A = rng.integers(-2, 3, (nwin[0] * nwin[1] * inner, nop)).astype(np.float64)
    MM = restated("MatrixMult")
    if n[0] == 1:
        nwins = len(np.arange(0, n[1] - nwin[1] + 1, nwin[1] - nover[1]))
        S = restated("Sliding2D")(MM(A), (nwins * nop, 1), (n[1], inner), nwin[1], nover[1], tapertype=tapertype)
    else:
        nw = [len(np.arange(0, n[a] - nwin[a] + 1, nwin[a] - nover[a])) for a in (0, 1)]
        S = restated("Sliding3D")(MM(A), (nw[0] * 2, nw[1] * 2, 1), (n[0], n[1], inner), nwin, nover, (2, 2, 1),
                                  tapertype=tapertype)
    M = dense_sliding(A, n, nwin, nover, tapertype, inner)
    assert S.shape == M.shape and np.count_nonzero(M) > 0
    D = np.stack([S.matvec(e) for e in np.eye(M.shape[1])], 1)
    Da = np.stack([S.rmatvec(e) for e in np.eye(M.shape[0])], 1)
    if tapertype in ("hanning", None) and max(nover) <= 3:
        np.testing.assert_array_equal(D, M)
        np.testing.assert_array_equal(Da, M.T)
    else:
        np.testing.assert_allclose(D, M, rtol=1e-14, atol=1e-14)
        np.testing.assert_allclose(Da, M.T, rtol=1e-14, atol=1e-14)


def test_restatement_argument_errors():
    MM, S2, S3 = restated("MatrixMult"), restated("Sliding2D"), restated("Sliding3D")
    A = MM(np.ones((8 * 5, 4)))
    S2(A, (12, 1), (22, 5), 8, 3)
    for dims, dimsd, nwin, nover in (((12, 1), (22, 5), 8, 8), ((12, 1), (7, 5), 8, 3), ((8, 1), (22, 5), 8, 3),
                                     ((12, 1), (22, 5), 8, 5)):
        with pytest.raises(ValueError):
            S2(A, dims, dimsd, nwin, nover)
    B = MM(np.ones((6 * 6 * 2, 4)))
    S3(B, (4, 4, 1), (9, 10, 2), (6, 6), (3, 3), (2, 2, 1))
    with pytest.raises(ValueError):
        S3(B, (4, 2, 1), (9, 10, 2), (6, 6), (3, 3), (2, 2, 1))


def test_library_tapers_and_design_are_the_restatement():
    """the host taper table and the design helpers of pylops_mpi_b200.local against the restatement"""
    import pylops_mpi_b200.local as L
    s2d = restated("Sliding2D")
    rs2, rs3 = sys.modules[s2d.__module__], sys.modules[restated("Sliding3D").__module__]
    for n, nwin, nover, tapertype in DEFS:
        if n[0] == 1:
            nw = len(L._slidingsteps(n[1], nwin[1], nover[1]))
            got = L._axis_tapers(nw, nwin[1], nover[1], tapertype, lambda t: 1.0)
            want = rs2.window_tapers(nw, 1, nwin[1], nover[1], tapertype)
            want = np.ones((nw, nwin[1])) if want is None else np.stack([t[:, 0] for t in want])
            np.testing.assert_array_equal(got, want)
            a = L.sliding2d_design((n[1], 7), nwin[1], nover[1], (3, 7))
            b = rs2.sliding2d_design((n[1], 7), nwin[1], nover[1], (3, 7))
        else:
            nw = [len(L._slidingsteps(n[a], nwin[a], nover[a])) for a in (0, 1)]
            t0, t1 = (L._axis_tapers(nw[a], nwin[a], nover[a], tapertype, lambda t: t[len(t) // 2]) for a in (0, 1))
            want = rs3.window_tapers(nw[0], nw[1], 1, nwin, nover, tapertype)
            if want is not None:
                got = (t0[:, None, :, None] * t1[None, :, None, :]).reshape(nw[0] * nw[1], *nwin)
                np.testing.assert_array_equal(got, np.stack([t[:, :, 0] for t in want]))
            a = L.sliding3d_design((*n, 7), nwin, nover, (2, 3, 7))
            b = rs3.sliding3d_design((*n, 7), nwin, nover, (2, 3, 7))
        assert a[0] == b[0] and a[1] == b[1]
        for u, v in zip(a[2] + a[3], b[2] + b[3]):
            for p, q in zip(u, v):
                np.testing.assert_array_equal(p, q)


def test_operator_argument_errors_before_any_device_work():
    """TypeError for an Op that is not a kernel operator, checked first; then pylops' ValueErrors, on a kernel
    operator by type that needs no device"""
    import pylops_mpi_b200 as pm
    L = pm.local

    def op(shape, kernel=True):
        base = L._KernelOperator if kernel else L.LocalOperator
        return type("Window", (base,), {"shape": shape, "dtype": np.float64})()

    with pytest.raises(TypeError):
        L.Sliding2D(op((8 * 5, 4), kernel=False), (12, 1), (22, 5), 8, 3)
    with pytest.raises(TypeError):
        L.Sliding2D(op((4, 8 * 5)).H, (12, 1), (22, 5), 8, 3)
    for dims, dimsd, nwin, nover in (((12, 1), (22, 5), 8, 8), ((12, 1), (7, 5), 8, 3), ((8, 1), (22, 5), 8, 3),
                                     ((12, 1), (22, 5), 8, 5), ((12, 1), (22, 6), 8, 3)):
        with pytest.raises(ValueError):
            L.Sliding2D(op((8 * 5, 4)), dims, dimsd, nwin, nover)
    with pytest.raises(TypeError):
        L.Sliding3D(op((6 * 6 * 2, 4), kernel=False), (4, 4, 1), (9, 10, 2), (6, 6), (3, 3), (2, 2, 1))
    for dims, nover in (((4, 2, 1), (3, 3)), ((4, 4, 1), (6, 3))):
        with pytest.raises(ValueError):
            L.Sliding3D(op((6 * 6 * 2, 4)), dims, (9, 10, 2), (6, 6), nover, (2, 2, 1))


def test_fixture_inventory():
    want = set()
    for c in CASES:
        k = mgs.key(*c)
        nm, nd = mgs.sizes(c)
        ex = mgs.exact(*c)
        for n in (("y", "ya", "yi", "yai") if ex else ("y", "ya")):
            a = GOLD[f"{k}/{n}"]
            assert a.dtype == (np.int32 if ex else np.float64)
            assert a.shape == (mgs.NG * (nd if n in ("y", "yi") else nm),)
            want.add(f"{k}/{n}")
    assert len(CASES) == 2 * 3 * 2 + 6 + 2 + 4
    assert {g for *_, g in CASES} == set(mgs.GEOMS)
    want |= {"flow/d", "flow/alpha", "flow/cond", "flow/spread"}
    want |= {f"flow/P{P}/{k}" for P in (1, 2, 3) for k in ("x", "iiter", "cost")}
    assert sorted(GOLD.files) == sorted(want)
    assert GOLD["flow/spread"].shape == (2,) and float(GOLD["flow/spread"].max()) < 1e-10
    for P in (1, 2, 3):
        assert int(GOLD[f"flow/P{P}/iiter"]) == mgs.FLOW_NITER


def restated_sections(c, dt):
    x, v = mgs.case_inputs(c, dt)
    nm, nd = mgs.sizes(c)
    S = mgs.make(c, dt, mgs.refshim_lib)
    y = np.concatenate([S.matvec(x[g * nm:(g + 1) * nm]) for g in range(mgs.NG)])
    ya = np.concatenate([S.rmatvec(v[g * nd:(g + 1) * nd]) for g in range(mgs.NG)])
    return y, ya


def case_id(c):
    return mgs.key(*c)[3:]


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_fixtures_follow_the_restatement_in_every_dtype(case):
    ex = mgs.exact(*case)
    for dt in mgs.DTYPES if ex else ("float64",):
        y, ya = restated_sections(case, dt)
        gy, gya = decode(GOLD, mgs.key(*case), dt, mgs.ENC if ex else 1)
        assert y.dtype == np.dtype(dt)
        np.testing.assert_array_equal(y, gy)
        np.testing.assert_array_equal(ya, gya)


def test_flow_inputs_regenerate():
    d, alpha = mgs.flow_inputs()
    np.testing.assert_array_equal(d, GOLD["flow/d"])
    assert alpha == float(GOLD["flow/alpha"])


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernels through the C ABI
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


def dev(a, dt=np.float64):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a, dtype=dt)).cuda()


def fold_ref(win, n0, n1, inner, nw, L, st, tap, dt):
    """b2_sliding's forward in NumPy, in the dtype dt and the restated order: win [nw0][nw1][L0][L1][inner]"""
    win = win.reshape(nw[0] * nw[1], L[0], L[1], inner).astype(dt)
    out = np.zeros((n0, n1, inner), dtype=dt)
    for i0 in range(nw[0]):
        part = np.zeros((L[0], n1, inner), dtype=dt)
        for i1 in range(nw[1]):
            w = i0 * nw[1] + i1
            v = win[w] if tap is None else tap[w].astype(dt)[:, :, None] * win[w]
            part[:, i1 * st[1]:i1 * st[1] + L[1]] += v
        out[i0 * st[0]:i0 * st[0] + L[0]] += part
    return out.ravel()


def unfold_ref(d, n0, n1, inner, nw, L, st, tap, dt):
    d = d.reshape(n0, n1, inner).astype(dt)
    parts = []
    for i0 in range(nw[0]):
        for i1 in range(nw[1]):
            v = d[i0 * st[0]:i0 * st[0] + L[0], i1 * st[1]:i1 * st[1] + L[1]]
            parts.append(v if tap is None else tap[i0 * nw[1] + i1].astype(dt)[:, :, None] * v)
    return np.concatenate([p.ravel() for p in parts])


def c_sliding(pm, x, y, n0, n1, nt, ni, nw0, nw1, l0, l1, s0, s1, tap, adjoint, code):
    L = pm._lib
    return L.lib.b2_sliding(L.ctx(), x, y, n0, n1, nt, ni, nw0, nw1, l0, l1, s0, s1, tap, adjoint, code, L.stream())


# (n0, n1), (nw0, nw1), (L0, L1), (s0, s1), nt, n_inner: 2-D, 3-D with uncovered traces, singleton windows, n_inner 2,
# more values than 2^16 CTAs of 256 threads
SLIDING_SHAPES = [((1, 22), (1, 3), (1, 8), (1, 5), 7, 1), ((9, 10), (2, 2), (6, 6), (3, 3), 5, 2),
                  ((1, 1), (1, 1), (1, 1), (1, 1), 3, 1), ((4, 6), (4, 6), (1, 1), (1, 1), 2, 2),
                  ((1, 300), (1, 36), (1, 16), (1, 8), 30000, 2), ((5, 5), (1, 2), (5, 3), (1, 2), 4, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("tapered", [True, False], ids=["taper", "notaper"])
def test_sliding_kernel_vs_dense_fold(pm, dt, tapered):
    rng = np.random.default_rng(7 + int(tapered))
    code = pm._lib.F32 if dt == np.float32 else pm._lib.F64
    for n, nw, L, st, nt, ni in SLIDING_SHAPES:
        inner = nt * ni
        tap = rng.uniform(0, 1, (nw[0] * nw[1], L[0], L[1])).astype(dt) if tapered else None
        tp = dev(tap, dt) if tapered else None
        nwv = nw[0] * nw[1] * L[0] * L[1] * inner
        ndv = n[0] * n[1] * inner
        # the fold matrix from the geometry: data x windows, in float64
        if ndv * nwv <= 4e6:
            F = np.zeros((ndv, nwv))
            t = np.ones((nw[0] * nw[1], L[0], L[1])) if tap is None else tap.astype(np.float64)
            for w in range(nw[0] * nw[1]):
                i0, i1 = divmod(w, nw[1])
                for j0 in range(L[0]):
                    for j1 in range(L[1]):
                        r = ((i0 * st[0] + j0) * n[1] + i1 * st[1] + j1) * inner + np.arange(inner)
                        c = ((w * L[0] + j0) * L[1] + j1) * inner + np.arange(inner)
                        F[r, c] = t[w, j0, j1]
        else:
            F = None
        for adjoint in (False, True):
            x = rng.standard_normal(ndv if adjoint else nwv).astype(dt)
            xd = dev(x, dt)
            args = (n[0], n[1], nt, ni, nw[0], nw[1], L[0], L[1], st[0], st[1],
                    None if tp is None else tp.data_ptr(), int(adjoint), code)
            got, guards, same = guarded_twice(lambda yp: c_sliding(pm, xd.data_ptr(), yp, *args),
                                              nwv if adjoint else ndv, dt, 3, offset=1)
            assert guards and same, (n, nw, adjoint)
            ref = (unfold_ref if adjoint else fold_ref)(x, n[0], n[1], inner, nw, L, st, tap, dt)
            np.testing.assert_array_equal(got, ref)
            if F is not None:
                M = F.T if adjoint else F
                np.testing.assert_allclose(got, M @ x.astype(np.float64), rtol=1e-5 if dt == np.float32 else 1e-13,
                                           atol=1e-5 if dt == np.float32 else 1e-13)


@pytest.mark.gpu
def test_sliding_kernel_error_codes_leave_y_untouched(pm):
    import torch
    L = pm._lib
    ARG, DT = 2002, 2001
    x = torch.ones(22 * 7, dtype=torch.float64, device="cuda")
    y = torch.full((3 * 8 * 7,), 3.5, dtype=torch.float64, device="cuda")
    base = dict(x=x.data_ptr(), y=y.data_ptr(), n0=1, n1=22, nt=7, ni=1, nw0=1, nw1=3, l0=1, l1=8, s0=1, s1=5,
                tap=None, adjoint=1, code=L.F64)
    big = 1 << 31
    cases = [(dict(x=None), ARG), (dict(y=None), ARG), (dict(y="x"), ARG), (dict(n0=0), ARG), (dict(n1=0), ARG),
             (dict(nt=0), ARG), (dict(ni=0), ARG), (dict(nw1=0), ARG), (dict(l1=0), ARG), (dict(s1=0), ARG),
             (dict(nw1=4), ARG), (dict(l1=23), ARG), (dict(s1=8), ARG), (dict(l0=2), ARG), (dict(nt=big), ARG),
             (dict(n1=big), ARG), (dict(nt=1 << 30, ni=1 << 30), ARG),
             (dict(code=L.C64), DT), (dict(code=L.C128), DT), (dict(code=L.BF16), DT), (dict(code=99), DT)]
    assert_rejected(lambda a: c_sliding(pm, *a.values()), base, cases, y)


def c_radon(pm, x, y, nt, ni, nhy, nhx, npy, npx, hy, hx, py, px, kind, interp, adjoint, code):
    L = pm._lib
    return L.lib.b2_radon(L.ctx(), x, y, nt, ni, nhy, nhx, npy, npx, hy, hx, py, px, kind, interp, adjoint, code,
                          L.stream())


def c_radon_windows(pm, x, y, nt, ni, n0, n1, nhy, nhx, npy, npx, hy, hx, py, px, kind, interp, nw0, nw1, s0, s1,
                    tap, adjoint, code):
    L = pm._lib
    return L.lib.b2_radon_windows(L.ctx(), x, y, nt, ni, n0, n1, nhy, nhx, npy, npx, hy, hx, py, px, kind, interp,
                                  nw0, nw1, s0, s1, tap, adjoint, code, L.stream())


def window_axes(kind, three, rng):
    hx = np.sort(rng.uniform(-8, 8, 6))
    px = {"linear": rng.uniform(-1.5, 1.5, 5), "parabolic": rng.uniform(-0.2, 0.2, 5),
          "hyperbolic": np.abs(rng.uniform(0, 2, 5))}[kind]
    if kind == "hyperbolic":
        px[0] = 0.0
    if not three:
        return None, hx, None, px
    hy = np.sort(rng.uniform(-6, 6, 4))
    py = rng.uniform(-1, 1, 2) * (0.2 if kind == "parabolic" else 1.0)
    return hy, hx, (np.abs(py) + 0.5 if kind == "hyperbolic" else py), px


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("interp", [True, False], ids=["interp", "nointerp"])
@pytest.mark.parametrize("kind", mgr_radon.KINDS)
@pytest.mark.parametrize("ndim", [2, 3], ids=["2d", "3d"])
def test_radon_windows_equals_per_window_route(pm, ndim, kind, interp, dt):
    """b2_radon_windows against b2_radon per window plus b2_sliding, bit for bit, real and complex, tapered or not"""
    import torch
    rng = np.random.default_rng(40 + 10 * ndim + 2 * mgr_radon.KINDS.index(kind) + int(interp))
    hy, hx, py, px = window_axes(kind, ndim == 3, rng)
    ax = [None if a is None else dev(a) for a in (hy, hx, py, px)]
    ptr = [None if a is None else a.data_ptr() for a in ax]
    nhy, npy = (1, 1) if hy is None else (len(hy), len(py))
    nhx, npx = len(hx), len(px)
    nt = 300
    (n0, nw0, s0) = (1, 1, 1) if ndim == 2 else (10, 3, 3)
    n1, nw1, s1 = 17, 3, 4                         # trace 16 past the last window
    nw = nw0 * nw1
    code = pm._lib.F32 if dt == np.float32 else pm._lib.F64
    kcode = mgr_radon.KINDS.index(kind)
    for ni in (1, 2):
        for tapered in (True, False):
            tap = dev(rng.uniform(0, 1, (nw, nhy, nhx)), dt) if tapered else None
            tptr = None if tap is None else tap.data_ptr()
            nm, nwd, nd = npy * npx * nt * ni, nhy * nhx * nt * ni, n0 * n1 * nt * ni
            work = torch.empty(nw * nwd, dtype=getattr(torch, np.dtype(dt).name), device="cuda")
            geo = (n0, n1, nt, ni, nw0, nw1, nhy, nhx, s0, s1, tptr)
            for adjoint in (False, True):
                x = dev(rng.standard_normal(nd if adjoint else nw * nm).astype(dt), dt)
                ref = torch.empty(nw * nm if adjoint else nd, dtype=x.dtype, device="cuda")
                if adjoint:
                    assert c_sliding(pm, x.data_ptr(), work.data_ptr(), *geo, 1, code) == 0
                for w in range(nw):
                    src, dst = (work[w * nwd:], ref[w * nm:]) if adjoint else (x[w * nm:], work[w * nwd:])
                    assert c_radon(pm, src.data_ptr(), dst.data_ptr(), nt, ni, nhy, nhx, npy, npx, *ptr, kcode,
                                   int(interp), int(adjoint), code) == 0
                if not adjoint:
                    assert c_sliding(pm, work.data_ptr(), ref.data_ptr(), *geo, 0, code) == 0
                got, guards, same = guarded_twice(
                    lambda yp: c_radon_windows(pm, x.data_ptr(), yp, nt, ni, n0, n1, nhy, nhx, npy, npx, *ptr, kcode,
                                               int(interp), nw0, nw1, s0, s1, tptr, int(adjoint), code),
                    ref.numel(), dt, 3)
                assert guards and same
                np.testing.assert_array_equal(got, host(ref), err_msg=f"ni={ni} tapered={tapered} adj={adjoint}")
                assert np.count_nonzero(got) > 0


@pytest.mark.gpu
def test_radon_windows_error_codes_leave_y_untouched(pm):
    import torch
    L = pm._lib
    ARG, DT = 2002, 2001
    nt, nh, npp = 10, 3, 4
    x = torch.ones(2 * npp * nt, dtype=torch.float64, device="cuda")
    y = torch.full((5 * nt,), 3.5, dtype=torch.float64, device="cuda")
    ax = torch.arange(4, dtype=torch.float64, device="cuda")
    base = dict(x=x.data_ptr(), y=y.data_ptr(), nt=nt, ni=1, n0=1, n1=5, nhy=1, nhx=nh, npy=1, npx=npp, hy=None,
                hx=ax.data_ptr(), py=None, px=ax.data_ptr(), kind=0, interp=1, nw0=1, nw1=2, s0=1, s1=2, tap=None,
                adjoint=0, code=L.F64)
    cases = [(dict(x=None), ARG), (dict(y=None), ARG), (dict(y="x"), ARG), (dict(hx=None), ARG),
             (dict(hy=ax.data_ptr()), ARG), (dict(nhy=2), ARG), (dict(nt=0), ARG), (dict(ni=3), ARG),
             (dict(kind=3), ARG), (dict(n1=0), ARG), (dict(n1=4), ARG), (dict(nw1=3), ARG), (dict(s1=0), ARG),
             (dict(nw0=0), ARG), (dict(n0=1 << 31), ARG), (dict(nt=1 << 30, n0=1 << 20, nw0=1 << 20), ARG),
             (dict(code=L.C64), DT), (dict(code=L.BF16), DT), (dict(code=99), DT)]
    assert_rejected(lambda a: c_radon_windows(pm, *a.values()), base, cases, y)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the operators
# ---------------------------------------------------------------------------------------------------------------
def device_lib(pm):
    return lambda name: getattr(pm.local, name)


def blockdiag(pm, ng, c, dt):
    return pm.MPIBlockDiag([mgs.make(c, dt, device_lib(pm)) for _ in range(ng)], dtype=dt)


def check_close(got, ref, bnd, k, dt):
    """got ~ ref: the float64 chain's error is within (k + 4) u of the sum of |terms| bnd, float32 once more"""
    tol = (k + 4) * U64 * bnd + (4 * k * U32 * bnd if dt == np.float32 else 0)
    err = np.abs(got - ref)
    assert np.all(err <= tol + 1e-300), f"max err {err.max():.3e}, worst ratio {np.max(err / (tol + 1e-300)):.3f}"


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_operator_vs_reference_fixtures(pm, case, P):
    """exact cases bit for bit in every dtype, the others in float64 and float32 under a rounding bound of the
    float64 fixture; the P ranks' sections as one rank's blocks"""
    ex = mgs.exact(*case)
    for dt in mgs.DTYPES if ex else ("float64", "float32"):
        x, v = mgs.case_inputs(case, dt)
        Op = blockdiag(pm, sum(rows_of(P, mgs.NG)), case, dt)
        S = Op.ops[0] if hasattr(Op, "ops") else None
        if S is not None:
            assert (S._fused is not None) == (case[0] == "radon")
        got = host((Op @ pm.DistributedArray.to_dist(x)).asarray())
        gota = host((Op.H @ pm.DistributedArray.to_dist(v)).asarray())
        assert got.dtype == np.dtype(dt) and gota.dtype == np.dtype(dt)
        if ex:
            gy, gya = decode(GOLD, mgs.key(*case), dt, mgs.ENC)
            np.testing.assert_array_equal(got, gy)
            np.testing.assert_array_equal(gota, gya)
            continue
        gy, gya = decode(GOLD, mgs.key(*case), "float64", 1)
        if dt == "float64":
            bx, bv = np.abs(x.astype(np.float64)), np.abs(v.astype(np.float64))
        else:
            bx, bv = np.abs(x).astype(np.float64), np.abs(v).astype(np.float64)
        So = mgs.make(case, "float64", mgs.refshim_lib)
        M = np.abs(np.stack([So.matvec(e) for e in np.eye(So.shape[1])], 1))
        nm, nd = mgs.sizes(case)
        k = max(int(np.count_nonzero(M, 1).max()), int(np.count_nonzero(M, 0).max()))
        rdt = np.float32 if dt == "float32" else np.float64
        bnd = np.concatenate([M @ bx[g * nm:(g + 1) * nm] for g in range(mgs.NG)])
        bnda = np.concatenate([M.T @ bv[g * nd:(g + 1) * nd] for g in range(mgs.NG)])
        check_close(got.astype(np.float64), gy, bnd, k, rdt)
        check_close(gota.astype(np.float64), gya, bnda, k, rdt)


@pytest.mark.gpu
@pytest.mark.parametrize("inner", ["radon2d", "radon3d", "matrix2d"])
def test_operator_dottest(pm, inner):
    from pylops_mpi_b200.utils.dottest import dottest
    rng = np.random.default_rng(8)
    L = pm.local
    if inner == "radon3d":
        t = np.arange(150) * 0.004
        R = L.Radon3D(t, np.arange(6) * 10.0, np.arange(8) * 10.0, np.linspace(-1e-3, 1e-3, 3),
                      np.linspace(-2e-3, 2e-3, 5), kind="parabolic")
        nw, dims, _, _ = L.sliding3d_design((15, 20, 150), (6, 8), (3, 4), (3, 5, 150))
        S = L.Sliding3D(R, dims, (15, 20, 150), (6, 8), (3, 4), (3, 5, 150))
    else:
        t = np.arange(300) * 0.004
        if inner == "radon2d":
            R = L.Radon2D(t, np.arange(32) * 12.5, np.linspace(0.0, 3000.0, 40), kind="hyperbolic")
            nop = (40, 300)
        else:
            R = L.MatrixMult(rng.standard_normal((32 * 300, 50)))
            nop = (5, 10)
        nw, dims, _, _ = L.sliding2d_design((150, 300), 32, 16, nop)
        S = L.Sliding2D(R, dims, (150, 300), 32, 16, tapertype="cosine")
    Op = pm.MPIBlockDiag([S, S])
    u = pm.DistributedArray.to_dist(rng.standard_normal(Op.shape[1]))
    v = pm.DistributedArray.to_dist(rng.standard_normal(Op.shape[0]))
    assert dottest(Op, u, v, rtol=1e-12)


@pytest.mark.gpu
def test_operator_attributes_and_paths(pm):
    L = pm.local
    t = np.arange(20) * 0.004
    R = L.Radon2D(t, np.arange(8) * 10.0, np.linspace(-1e-3, 1e-3, 4))
    S = L.Sliding2D(R, (12, 20), (22, 20), 8, 3, name="W")
    assert (S.dims, S.dimsd, S.shape) == ((12, 20), (22, 20), (440, 240))
    assert (S.nwin, S.nover, S.tapertype, S.name, S.dtype) == (8, 3, "hanning", "W", np.float64)
    assert S._fused is R
    M = L.MatrixMult(np.ones((8 * 20, 6), dtype=np.float32))
    S = L.Sliding2D(M, (18, 1), (22, 20), 8, 3, tapertype=None)
    assert S._fused is None and S.dtype == np.float32 and S.tapertype is None and S.name == "S"
    R3 = L.Radon3D(t, np.arange(6) * 10.0, np.arange(6) * 10.0, np.linspace(-1e-3, 1e-3, 2),
                   np.linspace(-1e-3, 1e-3, 3))
    S3 = L.Sliding3D(R3, (4, 6, 20), (9, 10, 20), (6, 6), (3, 3), (2, 3, 20), nproc=2)
    assert (S3.dims, S3.dimsd, S3.nwin, S3.nover, S3.nop, S3.name) == ((4, 6, 20), (9, 10, 20), (6, 6), (3, 3),
                                                                     (2, 3, 20), "P")
    assert S3._fused is R3
    with pytest.raises(TypeError):
        L.Sliding2D(R.H, (12, 20), (22, 20), 8, 3)
    with pytest.raises(TypeError):
        L.Sliding2D(R.H @ R, (12, 20), (22, 20), 8, 3)


# the _KernelOperator contract checks of test_local_apply.py, on sliding operators
# the inner operator's dtype and the result dtypes for data of dtype float32, float64, complex64, complex128
F32R, F64R = ("F32", "F32", "C64", "C128"), ("F64", "F64", "C128", "C128")
CONTRACT = {"Sliding2D-Radon2D": ("float64", F64R), "Sliding3D-Radon3D": ("float32", F32R),
            "Sliding2D-MatrixMult": ("float32", F32R), "Sliding3D-MatrixMult": ("float64", F64R)}


def make_contract(pm, name):
    rng = np.random.default_rng(5)
    L = pm.local
    t = np.arange(12) * 0.004
    dt = CONTRACT[name][0]
    if name == "Sliding2D-Radon2D":
        return L.Sliding2D(L.Radon2D(t, np.arange(6) * 10.0, np.linspace(-1e-3, 1e-3, 3), dtype=dt), (9, 12), (14, 12),
                           6, 2)
    if name == "Sliding3D-Radon3D":
        R = L.Radon3D(t, np.arange(4) * 10.0, np.arange(4) * 10.0, np.linspace(-1e-3, 1e-3, 2),
                      np.linspace(-1e-3, 1e-3, 2), dtype=dt)
        return L.Sliding3D(R, (4, 6, 12), (6, 8, 12), (4, 4), (2, 2), (2, 2, 12))
    if name == "Sliding2D-MatrixMult":
        return L.Sliding2D(L.MatrixMult(rng.standard_normal((6 * 5, 4)).astype(dt)), (12, 1), (14, 5), 6, 2,
                           tapertype="cosine")
    return L.Sliding3D(L.MatrixMult(rng.standard_normal((4 * 4 * 3, 4)).astype(dt)), (4, 6, 1), (6, 8, 3), (4, 4),
                       (2, 2), (2, 2, 1))

CHECKS = ["test_result_dtype", "test_out_equals_out_none", "test_complex_data_equals_its_parts",
          "test_complex_into_real_out_warns_and_keeps_the_real_part", "test_wrong_length_raises",
          "test_direct_out_allocates_nothing", "test_graph_safe_by_type"]


@pytest.mark.gpu
@pytest.mark.parametrize("check", CHECKS)
@pytest.mark.parametrize("name", list(CONTRACT))
def test_kernel_operator_contract(pm, monkeypatch, name, check):
    """each check of test_local_apply.py, run on the sliding operators through its own registry"""
    import test_local_apply as tla
    result = {name: tuple(getattr(tla, d) for d in CONTRACT[name][1])}
    monkeypatch.setattr(tla, "RESULT", result)
    monkeypatch.setattr(tla, "make", lambda pm_, n: make_contract(pm_, n))
    fn = getattr(tla, check)
    if check in ("test_result_dtype", "test_complex_data_equals_its_parts", "test_wrong_length_raises"):
        for adjoint in (False, True):
            fn(pm, name, adjoint)
    elif check == "test_out_equals_out_none":
        for adjoint in (False, True):
            for xdt in (tla.F32, tla.C128):
                fn(pm, name, adjoint, xdt)
    else:
        fn(pm, name)


@pytest.mark.gpu
@pytest.mark.parametrize("inner", ["radon", "matrix"])
def test_cgls_graph_replay_matches_step_loop(pm, inner):
    rng = np.random.default_rng(12)
    L = pm.local
    t = np.arange(64) * 0.004
    if inner == "radon":
        Op1 = L.Radon2D(t, np.arange(12) * 10.0, np.linspace(-1e-3, 1e-3, 21))
        nop = (21, 64)
    else:
        Op1 = L.MatrixMult(rng.standard_normal((12 * 64, 40)))
        nop = (40, 1)
    nw, dims, _, _ = L.sliding2d_design((30, 64), 12, 6, nop)
    Op = pm.MPIBlockDiag([L.Sliding2D(Op1, dims, (30, 64), 12, 6) for _ in range(2)])
    y = Op @ pm.DistributedArray.to_dist(rng.standard_normal(Op.shape[1]))
    assert_cgls_replay_matches_steps(pm, Op, y, pm.DistributedArray.to_dist(np.zeros(Op.shape[1])), 25, 20)


def flow_tolerance():
    """(x, cost) relative tolerances of the flow, as test_radon's: 100 times the 4-ulp jitter spread of the
    reference's own run, and no less than 10 cond 2^-53"""
    floor = 10 * float(GOLD["flow/cond"]) * 2.0 ** -53
    return tuple(max(100 * float(s), floor) for s in GOLD["flow/spread"])


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
def test_local_denoising_fista_vs_reference(pm, P):
    alpha = float(GOLD["flow/alpha"])
    Op = pm.MPIBlockDiag([mgs.flow_ops(device_lib(pm)) for r in rows_of(P, mgs.FLOW_NG) for _ in range(r)])
    x0 = pm.DistributedArray.to_dist(np.zeros(Op.shape[1]))
    x, iiter, cost = pm.fista(Op, pm.DistributedArray.to_dist(GOLD["flow/d"]), x0, niter=mgs.FLOW_NITER,
                              eps=mgs.FLOW_EPS, alpha=alpha, tol=1e-10)
    assert iiter == int(GOLD[f"flow/P{P}/iiter"])
    xtol, ctol = flow_tolerance()
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"flow/P{P}/cost"], rtol=ctol)
    gx = GOLD[f"flow/P{P}/x"]
    np.testing.assert_allclose(host(x.asarray()), gx, rtol=0, atol=xtol * np.abs(gx).max())


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [1, 2])
def test_multi_rank_fixtures(nproc):
    needs_gpus(nproc)
    run_on_ranks("test_sliding", nproc)


def on_ranks(pm, comm):
    """each rank's MPIBlockDiag of sliding operators against its slice of the gathered exact fixtures, and the fista
    flow against its fixture"""
    rank, P = comm.Get_rank(), comm.Get_size()

    def split(n_per, ng):
        rows = rows_of(P, ng)
        lo, hi = sum(rows[:rank]) * n_per, sum(rows[:rank + 1]) * n_per
        return [(r * n_per,) for r in rows], slice(lo, hi), rows[rank]

    for case in mgs.cases():
        if not mgs.exact(*case):
            continue
        nm, nd = mgs.sizes(case)
        lsm, slm, ng = split(nm, mgs.NG)
        lsd, sld, _ = split(nd, mgs.NG)
        for dt in mgs.DTYPES:
            x, v = mgs.case_inputs(case, dt)
            Op = blockdiag(pm, ng, case, dt)
            gy, gya = decode(GOLD, mgs.key(*case), dt, mgs.ENC)
            name = f"{mgs.key(*case)}/{dt}"
            np.testing.assert_array_equal(host((Op @ pm.DistributedArray.to_dist(x, local_shapes=lsm)).local_array),
                                          gy[sld], err_msg=f"[rank {rank}] {name}/y")
            np.testing.assert_array_equal(host((Op.H @ pm.DistributedArray.to_dist(v, local_shapes=lsd)).local_array),
                                          gya[slm], err_msg=f"[rank {rank}] {name}/ya")

    nd = mgs.FLOW_N * mgs.FLOW_NT
    S = mgs.flow_ops(device_lib(pm))
    nm = S.shape[1]
    lsd, sld, ng = split(nd, mgs.FLOW_NG)
    lsm, slm, _ = split(nm, mgs.FLOW_NG)
    Op = pm.MPIBlockDiag([mgs.flow_ops(device_lib(pm)) for _ in range(ng)])
    d = pm.DistributedArray.to_dist(GOLD["flow/d"], local_shapes=lsd)
    x0 = pm.DistributedArray.to_dist(np.zeros(mgs.FLOW_NG * nm), local_shapes=lsm)
    x, iiter, cost = pm.fista(Op, d, x0, niter=mgs.FLOW_NITER, eps=mgs.FLOW_EPS, alpha=float(GOLD["flow/alpha"]),
                              tol=1e-10)
    assert iiter == int(GOLD[f"flow/P{P}/iiter"])
    xtol, ctol = flow_tolerance()
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"flow/P{P}/cost"], rtol=ctol, err_msg=f"[rank {rank}] cost")
    gx = GOLD[f"flow/P{P}/x"]
    np.testing.assert_allclose(host(x.local_array), gx[slm], rtol=0, atol=xtol * np.abs(gx).max(),
                               err_msg=f"[rank {rank}] x")
