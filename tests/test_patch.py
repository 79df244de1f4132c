"""Rank-local Sliding1D / Patch2D / Patch3D (pylops.signalprocessing.Sliding1D / Patch2D / Patch3D inside
MPIBlockDiag): windows along the traces and the samples of a section, one inner operator per window, tapered and
overlap-added in the nested chain's order (over i0, of the sum over i1, of the sum over i2, all ascending).

CPU: refshim's restatement (tests/golden/refshim/pylops/signalprocessing/patch2d.py, patch3d.py, sliding1d.py) against
a dense matrix built directly from the definition, argument errors, the library's per-axis tapers and design helpers
against the restated full tapers, and the fixtures of tests/golden/patch_golden.npz (made by make_golden_patch.py: the
reference's MPIBlockDiag and FISTA over the restatement).  GPU: the b2_patch and b2_radon_patches kernels through the
C ABI and the operators through the public interface."""
import itertools
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_patch as mgp  # noqa: E402
import make_golden_radon as mgr_radon  # noqa: E402
from fixture_codec import decode, rows_of  # noqa: E402
from op_checks import (assert_cgls_replay_matches_steps, assert_rejected, guarded_twice, host,  # noqa: E402
                       needs_gpus, run_on_ranks)
from test_sliding import check_close, rise, window_axes  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "patch_golden.npz"), allow_pickle=False)
CASES = mgp.cases()


# ---------------------------------------------------------------------------------------------------------------
# the definition, built directly
# ---------------------------------------------------------------------------------------------------------------
def axis_taper(nwin, nover, tapertype):
    tap = np.ones(nwin)
    if tapertype is not None:
        r = rise(nover, tapertype)
        tap[:len(r)] = r
        tap[nwin - len(r):] = r[::-1]
    return tap


def full_tapers(n, nwin, nover, tapertype):
    """(starts per axis, {window index tuple: full taper}) of the definition: Sliding1D's edge samples set to 1;
    Patch2D's / Patch3D's edge rows / columns set to the middle ones (one window: the trailing ones only), Patch3D
    constant along t"""
    K = len(n)
    starts = [np.arange(0, n[a] - nwin[a] + 1, nwin[a] - nover[a]) for a in range(K)]
    axes = []
    for a in range(K):
        tapered = tapertype is not None and not (K == 3 and a == 2)
        base = axis_taper(nwin[a], nover[a], tapertype if tapered else None)
        edge = 1.0 if K == 1 else base[nwin[a] // 2]
        t = np.tile(base, (len(starts[a]), 1))
        if len(starts[a]) > 1:
            t[0, :nover[a]] = edge
        t[-1, nwin[a] - nover[a]:] = edge
        axes.append(t)
    taps = {}
    for idx in itertools.product(*[range(len(s)) for s in starts]):
        full = np.ones(())
        for a, i in enumerate(idx):
            full = np.multiply.outer(full, axes[a][i])
        taps[idx] = full
    return starts, taps


def dense_patches(A, n, nwin, nover, tapertype):
    starts, taps = full_tapers(n, nwin, nover, tapertype)
    nwins = [len(s) for s in starts]
    nm = A.shape[1]
    M = np.zeros((int(np.prod(n)), int(np.prod(nwins)) * nm))
    for idx, tap in taps.items():
        w = int(np.ravel_multi_index(idx, nwins))
        for j in itertools.product(*[range(v) for v in nwin]):
            r = int(np.ravel_multi_index(tuple(s[i] + jj for s, i, jj in zip(starts, idx, j)), n))
            M[r, w * nm:(w + 1) * nm] += tap[j] * A[int(np.ravel_multi_index(j, nwin))]
    return M


DEFS = [((22,), (8,), (3,), "hanning"), ((21,), (10,), (4,), "cosine"), ((8,), (8,), (3,), None),
        ((22, 20), (8, 8), (3, 3), "hanning"), ((8, 20), (8, 8), (3, 3), "hanning"),
        ((16, 20), (8, 8), (0, 3), "hanning"), ((21, 19), (10, 8), (4, 3), "cosinesquare"),
        ((9, 10, 14), (6, 6, 8), (3, 3, 3), "hanning"), ((6, 10, 16), (6, 6, 8), (3, 3, 0), "cosine"),
        ((9, 9, 9), (6, 6, 4), (3, 3, 2), None)]


def restated_op(A, n, nwin, nover, tapertype):
    MM = mgp.restated("MatrixMult")(A)
    nm = A.shape[1]
    nwins = [len(np.arange(0, n[a] - nwin[a] + 1, nwin[a] - nover[a])) for a in range(len(n))]
    if len(n) == 1:
        return mgp.restated("Sliding1D")(MM, nwins[0] * nm, n[0], nwin[0], nover[0], tapertype=tapertype)
    nop = (1,) * (len(n) - 1) + (nm,)
    dims = tuple(w * p for w, p in zip(nwins, nop))
    return mgp.restated(mgp.CLASS[len(n)])(MM, dims, n, nwin, nover, nop, tapertype=tapertype)


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", DEFS, ids=[f"{d[0]}-{d[1]}-{d[2]}-{d[3]}" for d in DEFS])
def test_restatement_is_the_dense_definition(geom):
    n, nwin, nover, tapertype = geom
    rng = np.random.default_rng(sum(n) + sum(nwin))
    A = rng.integers(-2, 3, (int(np.prod(nwin)), 3)).astype(np.float64)
    S = restated_op(A, n, nwin, nover, tapertype)
    M = dense_patches(A, n, nwin, nover, tapertype)
    assert S.shape == M.shape and np.count_nonzero(M) > 0
    D = np.stack([S.matvec(e) for e in np.eye(M.shape[1])], 1)
    Da = np.stack([S.rmatvec(e) for e in np.eye(M.shape[0])], 1)
    np.testing.assert_allclose(D, M, rtol=1e-14, atol=1e-14)
    np.testing.assert_allclose(Da, M.T, rtol=1e-14, atol=1e-14)


def test_restatement_argument_errors():
    MM, P2, P3, S1 = (mgp.restated(n) for n in ("MatrixMult", "Patch2D", "Patch3D", "Sliding1D"))
    A = MM(np.ones((8 * 8, 4)))
    P2(A, (6, 6), (22, 20), (8, 8), (3, 3), (2, 2))
    for dims, dimsd, nwin, nover in (((6, 4), (22, 20), (8, 8), (3, 3)), ((6, 6), (7, 20), (8, 8), (3, 3)),
                                     ((6, 6), (22, 20), (8, 8), (8, 3)), ((6, 6), (22, 20), (8, 8), (5, 3))):
        with pytest.raises(ValueError):
            P2(A, dims, dimsd, nwin, nover, (2, 2))
    with pytest.raises(NotImplementedError):
        P2(A, (6, 6), (22, 20), (8, 8), (3, 3), (2, 2), scalings=np.ones(9))
    B = MM(np.ones((6 * 6 * 8, 2)))
    P3(B, (2, 2, 4), (9, 10, 14), (6, 6, 8), (3, 3, 3), (1, 1, 2))
    with pytest.raises(ValueError):
        P3(B, (2, 2, 2), (9, 10, 14), (6, 6, 8), (3, 3, 3), (1, 1, 2))
    C = MM(np.ones((8, 3)))
    S1(C, 9, 22, 8, 3)
    with pytest.raises(ValueError):
        S1(C, 12, 22, 8, 3)


def lib_taper_product(L, n, nwin, nover, tapertype):
    nwins = [len(L._slidingsteps(n[a], nwin[a], nover[a])) for a in range(len(n))]
    taps = L._patch_tapers(nwins, nwin, nover, tapertype)
    k = 3 - len(n)
    full = {}
    if tapertype is None:
        return nwins, taps, full
    for idx in itertools.product(*[range(w) for w in nwins]):
        t = np.ones(())
        for a, tab in enumerate(taps[k:]):
            t = np.multiply.outer(t, tab[idx[a]])     # ((t0 * t1) * t2) in float64, as the kernels form it
        full[idx] = t
    return nwins, taps, full


def test_library_tapers_and_design_are_the_restatement():
    """the product of the library's per-axis tables against the restated full pylops taper, bit for bit, and the
    design helpers against the restatement"""
    import pylops_mpi_b200.local as L
    for n, nwin, nover, tapertype in DEFS:
        nwins, taps, full = lib_taper_product(L, n, nwin, nover, tapertype)
        A = np.ones((int(np.prod(nwin)), 1))
        S = restated_op(A, n, nwin, nover, tapertype)
        if tapertype is None:
            assert S.taps is None and all(t is None for t in taps)
        else:
            assert len(S.taps) == int(np.prod(nwins))
            for idx, t in full.items():
                want = S.taps[int(np.ravel_multi_index(idx, nwins))]
                assert want.shape == t.shape
                np.testing.assert_array_equal(t, want, err_msg=f"{n} {nwin} {nover} {tapertype} {idx}")
        nop = (3,) * len(n)
        mod = sys.modules[type(S).__module__]
        if len(n) == 1:
            a = L.sliding1d_design(n[0], nwin[0], nover[0], nop[0])
            b = mod.sliding1d_design(n[0], nwin[0], nover[0], nop[0])
            assert a[:2] == b[:2]
            pairs = [(a[2], b[2]), (a[3], b[3])]
        else:
            design = "patch2d_design" if len(n) == 2 else "patch3d_design"
            a = getattr(L, design)(n, nwin, nover, nop)
            b = getattr(mod, design)(n, nwin, nover, nop)
            assert tuple(a[0]) == tuple(b[0]) and tuple(a[1]) == tuple(b[1])
            pairs = list(zip(a[2] + a[3], b[2] + b[3]))
        for u, v in pairs:
            for p, q in zip(u, v):
                np.testing.assert_array_equal(p, q)


def test_operator_argument_errors_before_any_device_work():
    """TypeError for an Op that is not a kernel operator, checked first; then pylops' errors, on a kernel operator by
    type that needs no device"""
    import pylops_mpi_b200 as pm
    L = pm.local

    def op(shape, kernel=True):
        base = L._KernelOperator if kernel else L.LocalOperator
        return type("Window", (base,), {"shape": shape, "dtype": np.float64})()

    P2 = ((6, 6), (22, 20), (8, 8), (3, 3), (2, 2))
    with pytest.raises(TypeError):
        L.Patch2D(op((64, 4), kernel=False), *P2)
    with pytest.raises(TypeError):
        L.Patch2D(op((4, 64)).H, *P2)
    with pytest.raises(NotImplementedError, match="scalings"):
        L.Patch2D(op((64, 4)), *P2, scalings=np.ones(9))
    for dims, dimsd, nwin, nover, nop in (((6, 4), (22, 20), (8, 8), (3, 3), (2, 2)),
                                          ((6, 6), (7, 20), (8, 8), (3, 3), (2, 2)),
                                          ((6, 6), (22, 20), (8, 8), (8, 3), (2, 2)),
                                          ((6, 6), (22, 20), (8, 8), (3, -1), (2, 2)),
                                          ((6, 6), (22, 20), (8, 8), (5, 3), (2, 2)),
                                          ((6, 6), (22, 23), (8, 8), (3, 3), (2, 2)),
                                          ((6, 6), (22, 20), (8, 8), (3, 3), (2, 3))):
        with pytest.raises(ValueError):
            L.Patch2D(op((64, 4)), dims, dimsd, nwin, nover, nop)
    with pytest.raises(ValueError):
        L.Patch2D(op((63, 4)), *P2)
    with pytest.raises(TypeError):
        L.Patch3D(op((6 * 6 * 8, 2), kernel=False), (2, 2, 4), (9, 10, 14), (6, 6, 8), (3, 3, 3), (1, 1, 2))
    for dims, nover in (((2, 2, 2), (3, 3, 3)), ((2, 2, 4), (3, 3, 5))):
        with pytest.raises(ValueError):
            L.Patch3D(op((6 * 6 * 8, 2)), dims, (9, 10, 14), (6, 6, 8), nover, (1, 1, 2))
    with pytest.raises(TypeError):
        L.Sliding1D(op((8, 3), kernel=False), 9, 22, 8, 3)
    for dim, dimd, nwin, nover in ((12, 22, 8, 3), (9, 7, 8, 3), (9, 22, 8, 8), (9, 22, 8, 5)):
        with pytest.raises(ValueError):
            L.Sliding1D(op((8, 3)), dim, dimd, nwin, nover)
    with pytest.raises(ValueError):
        L.Sliding1D(op((7, 3)), 9, 22, 8, 3)


def test_fixture_inventory():
    want = set()
    for c in CASES:
        k = mgp.key(*c)
        nm, nd = mgp.sizes(c)
        ex = mgp.exact(*c)
        for n in (("y", "ya", "yi", "yai") if ex else ("y", "ya")):
            a = GOLD[f"{k}/{n}"]
            assert a.dtype == (np.int32 if ex else np.float64)
            assert a.shape == (mgp.NG * (nd if n in ("y", "yi") else nm),)
            want.add(f"{k}/{n}")
    assert len(CASES) == 2 * 3 * 2 + 5 + 2 + 5
    assert {c[3] for c in CASES} == set(mgp.GEOMS)
    want |= {"flow/d", "flow/alpha", "flow/cond", "flow/spread"}
    want |= {f"flow/P{P}/{k}" for P in (1, 2, 3) for k in ("x", "iiter", "cost")}
    assert sorted(GOLD.files) == sorted(want)
    assert GOLD["flow/spread"].shape == (2,) and float(GOLD["flow/spread"].max()) < 1e-10
    for P in (1, 2, 3):
        assert int(GOLD[f"flow/P{P}/iiter"]) == mgp.FLOW_NITER


def case_id(c):
    return mgp.key(*c)[3:]


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_fixtures_follow_the_restatement_in_every_dtype(case):
    ex = mgp.exact(*case)
    nm, nd = mgp.sizes(case)
    for dt in mgp.DTYPES if ex else ("float64",):
        x, v = mgp.case_inputs(case, dt)
        S = mgp.make(case, dt, mgp.refshim_lib)
        y = np.concatenate([S.matvec(x[g * nm:(g + 1) * nm]) for g in range(mgp.NG)])
        ya = np.concatenate([S.rmatvec(v[g * nd:(g + 1) * nd]) for g in range(mgp.NG)])
        gy, gya = decode(GOLD, mgp.key(*case), dt, mgp.ENC if ex else 1)
        assert y.dtype == np.dtype(dt)
        np.testing.assert_array_equal(y, gy)
        np.testing.assert_array_equal(ya, gya)


def test_flow_inputs_regenerate():
    d, alpha = mgp.flow_inputs()
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


def c_patch(pm, x, y, n0, n1, nt, ni, nw0, nw1, nw2, l0, l1, l2, s0, s1, s2, t0, t1, t2, adjoint, code):
    L = pm._lib
    return L.lib.b2_patch(L.ctx(), x, y, n0, n1, nt, ni, nw0, nw1, nw2, l0, l1, l2, s0, s1, s2, t0, t1, t2, adjoint,
                          code, L.stream())


def tap_of(taps, g, w, j, dt):
    """(T)((t0 * t1) * t2) of window w = (i0, i1, i2) at window sample j, the missing tables 1"""
    v = 1.0
    for a in range(3):
        if taps[a] is not None:
            v = v * taps[a][w[a], j[a]]
    return dt(v)


def fold_ref(win, n, nw, L, st, ni, taps, dt):
    """b2_patch's forward in NumPy, in the dtype dt and the chain's order: win [nw0][nw1][nw2][L0][L1][L2][ni]"""
    win = win.reshape(*nw, *L, ni).astype(dt)
    out = np.zeros((*n, ni), dtype=dt)
    for a, b, s in itertools.product(*[range(v) for v in n]):
        acc = dt(0)
        for i0 in range(nw[0]):
            if not 0 <= a - i0 * st[0] < L[0]:
                continue
            p1 = dt(0)
            for i1 in range(nw[1]):
                if not 0 <= b - i1 * st[1] < L[1]:
                    continue
                p2 = dt(0)
                for i2 in range(nw[2]):
                    j = (a - i0 * st[0], b - i1 * st[1], s - i2 * st[2])
                    if not 0 <= j[2] < L[2]:
                        continue
                    v = win[i0, i1, i2, j[0], j[1], j[2]]
                    if any(t is not None for t in taps):
                        v = tap_of(taps, None, (i0, i1, i2), j, dt) * v
                    p2 = p2 + v
                p1 = p1 + p2
            acc = acc + p1
        out[a, b, s] = acc
    return out.ravel()


def unfold_ref(d, n, nw, L, st, ni, taps, dt):
    d = d.reshape(*n, ni).astype(dt)
    out = np.zeros((*nw, *L, ni), dtype=dt)
    for w in itertools.product(*[range(v) for v in nw]):
        for j in itertools.product(*[range(v) for v in L]):
            v = d[w[0] * st[0] + j[0], w[1] * st[1] + j[1], w[2] * st[2] + j[2]]
            if any(t is not None for t in taps):
                v = tap_of(taps, None, w, j, dt) * v
            out[w + j] = v
    return out.ravel()


# (n0, n1, nt), (nw0, nw1, nw2), (L0, L1, L2), (s0, s1, s2), n_inner: Sliding1D, Patch2D with uncovered traces and
# samples, Patch3D, a single window, n_inner 2
PATCH_SHAPES = [((1, 1, 22), (1, 1, 3), (1, 1, 8), (1, 1, 5), 1), ((1, 22, 20), (1, 3, 3), (1, 8, 8), (1, 5, 5), 2),
                ((9, 10, 14), (2, 2, 2), (6, 6, 8), (3, 3, 5), 1), ((1, 8, 20), (1, 1, 2), (1, 8, 8), (1, 1, 8), 2),
                ((5, 5, 7), (1, 2, 3), (5, 3, 3), (1, 2, 2), 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("tapered", [True, False], ids=["taper", "notaper"])
def test_patch_kernel_vs_dense_fold(pm, dt, tapered):
    rng = np.random.default_rng(17 + int(tapered))
    code = pm._lib.F32 if dt == np.float32 else pm._lib.F64
    for n, nw, L, st, ni in PATCH_SHAPES:
        taps = [rng.uniform(0, 1, (nw[a], L[a])) if tapered and (a == 2 or n[a] > 1) else None for a in range(3)]
        tps = [None if t is None else dev(t) for t in taps]
        tpp = [None if t is None else t.data_ptr() for t in tps]
        nwv, ndv = int(np.prod(nw) * np.prod(L)) * ni, int(np.prod(n)) * ni
        for adjoint in (False, True):
            x = rng.standard_normal(ndv if adjoint else nwv).astype(dt)
            xd = dev(x, dt)
            args = (*n, ni, *nw, *L, *st, *tpp, int(adjoint), code)
            got, guards, same = guarded_twice(lambda yp: c_patch(pm, xd.data_ptr(), yp, *args),
                                              nwv if adjoint else ndv, dt, 3, offset=1)
            assert guards and same, (n, nw, adjoint)
            ref = (unfold_ref if adjoint else fold_ref)(x, n, nw, L, st, ni, taps, dt)
            np.testing.assert_array_equal(got, ref, err_msg=f"{n} {nw} adj={adjoint}")


@pytest.mark.gpu
def test_patch_kernel_error_codes_leave_y_untouched(pm):
    import torch
    L = pm._lib
    ARG, DT = 2002, 2001
    x = torch.ones(22 * 20, dtype=torch.float64, device="cuda")
    y = torch.full((9 * 64,), 3.5, dtype=torch.float64, device="cuda")
    base = dict(x=x.data_ptr(), y=y.data_ptr(), n0=1, n1=22, nt=20, ni=1, nw0=1, nw1=3, nw2=3, l0=1, l1=8, l2=8,
                s0=1, s1=5, s2=5, t0=None, t1=None, t2=None, adjoint=1, code=L.F64)
    big = 1 << 31
    cases = [(dict(x=None), ARG), (dict(y=None), ARG), (dict(y="x"), ARG), (dict(nt=0), ARG), (dict(ni=0), ARG),
             (dict(nw2=0), ARG), (dict(l2=0), ARG), (dict(s2=0), ARG), (dict(nw2=4), ARG), (dict(l2=21), ARG),
             (dict(s2=7), ARG), (dict(nt=big), ARG), (dict(nt=1 << 30, ni=1 << 30), ARG),
             (dict(code=L.C64), DT), (dict(code=L.BF16), DT), (dict(code=99), DT)]
    assert_rejected(lambda a: c_patch(pm, *a.values()), base, cases, y)


def c_radon(pm, x, y, nt, ni, nhy, nhx, npy, npx, hy, hx, py, px, kind, interp, adjoint, code):
    L = pm._lib
    return L.lib.b2_radon(L.ctx(), x, y, nt, ni, nhy, nhx, npy, npx, hy, hx, py, px, kind, interp, adjoint, code,
                          L.stream())


def c_radon_patches(pm, x, y, nt, ni, n0, n1, ns, nhy, nhx, npy, npx, hy, hx, py, px, kind, interp, nw0, nw1, nw2,
                    s0, s1, s2, t0, t1, t2, adjoint, code):
    L = pm._lib
    return L.lib.b2_radon_patches(L.ctx(), x, y, nt, ni, n0, n1, ns, nhy, nhx, npy, npx, hy, hx, py, px, kind,
                                  interp, nw0, nw1, nw2, s0, s1, s2, t0, t1, t2, adjoint, code, L.stream())


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("interp", [True, False], ids=["interp", "nointerp"])
@pytest.mark.parametrize("kind", mgr_radon.KINDS)
@pytest.mark.parametrize("ndim", [2, 3], ids=["2d", "3d"])
def test_radon_patches_equals_per_patch_route(pm, ndim, kind, interp, dt):
    """b2_radon_patches against b2_radon per patch plus b2_patch, bit for bit, real and complex, tapered or not"""
    import torch
    rng = np.random.default_rng(140 + 10 * ndim + 2 * mgr_radon.KINDS.index(kind) + int(interp))
    hy, hx, py, px = window_axes(kind, ndim == 3, rng)
    ax = [None if a is None else dev(a) for a in (hy, hx, py, px)]
    ptr = [None if a is None else a.data_ptr() for a in ax]
    nhy, npy = (1, 1) if hy is None else (len(hy), len(py))
    nhx, npx = len(hx), len(px)
    nt, ns, nw2, s2 = 300, 700, 3, 170                 # samples 640 .. 699 past the last patch
    (n0, nw0, s0) = (1, 1, 1) if ndim == 2 else (10, 3, 3)
    n1, nw1, s1 = 17, 3, 4                         # trace 16 past the last patch
    nw = nw0 * nw1 * nw2
    code = pm._lib.F32 if dt == np.float32 else pm._lib.F64
    kcode = mgr_radon.KINDS.index(kind)
    for ni in (1, 2):
        for tapered in (True, False):
            taps = [dev(rng.uniform(0, 1, (w, l))) if tapered and (a > 0 or ndim == 3) else None
                    for a, (w, l) in enumerate(((nw0, nhy), (nw1, nhx), (nw2, nt)))]
            tpp = [None if t is None else t.data_ptr() for t in taps]
            nm, nwd, nd = npy * npx * nt * ni, nhy * nhx * nt * ni, n0 * n1 * ns * ni
            work = torch.empty(nw * nwd, dtype=getattr(torch, np.dtype(dt).name), device="cuda")
            geo = (n0, n1, ns, ni, nw0, nw1, nw2, nhy, nhx, nt, s0, s1, s2, *tpp)
            for adjoint in (False, True):
                x = dev(rng.standard_normal(nd if adjoint else nw * nm).astype(dt), dt)
                ref = torch.empty(nw * nm if adjoint else nd, dtype=x.dtype, device="cuda")
                if adjoint:
                    assert c_patch(pm, x.data_ptr(), work.data_ptr(), *geo, 1, code) == 0
                for w in range(nw):
                    src, dst = (work[w * nwd:], ref[w * nm:]) if adjoint else (x[w * nm:], work[w * nwd:])
                    assert c_radon(pm, src.data_ptr(), dst.data_ptr(), nt, ni, nhy, nhx, npy, npx, *ptr, kcode,
                                   int(interp), int(adjoint), code) == 0
                if not adjoint:
                    assert c_patch(pm, work.data_ptr(), ref.data_ptr(), *geo, 0, code) == 0
                got, guards, same = guarded_twice(
                    lambda yp: c_radon_patches(pm, x.data_ptr(), yp, nt, ni, n0, n1, ns, nhy, nhx, npy, npx, *ptr,
                                               kcode, int(interp), nw0, nw1, nw2, s0, s1, s2, *tpp, int(adjoint),
                                               code),
                    ref.numel(), dt, 3)
                assert guards and same
                np.testing.assert_array_equal(got, host(ref), err_msg=f"ni={ni} tapered={tapered} adj={adjoint}")
                assert np.count_nonzero(got) > 0


@pytest.mark.gpu
def test_radon_patches_error_codes_leave_y_untouched(pm):
    import torch
    L = pm._lib
    ARG, DT = 2002, 2001
    nt, nh, npp = 10, 3, 4
    x = torch.ones(4 * npp * nt, dtype=torch.float64, device="cuda")
    y = torch.full((5 * 20,), 3.5, dtype=torch.float64, device="cuda")
    ax = torch.arange(4, dtype=torch.float64, device="cuda")
    base = dict(x=x.data_ptr(), y=y.data_ptr(), nt=nt, ni=1, n0=1, n1=5, ns=20, nhy=1, nhx=nh, npy=1, npx=npp,
                hy=None, hx=ax.data_ptr(), py=None, px=ax.data_ptr(), kind=0, interp=1, nw0=1, nw1=2, nw2=2, s0=1,
                s1=2, s2=10, t0=None, t1=None, t2=None, adjoint=0, code=L.F64)
    cases = [(dict(x=None), ARG), (dict(y=None), ARG), (dict(y="x"), ARG), (dict(hx=None), ARG),
             (dict(nt=0), ARG), (dict(ni=3), ARG), (dict(kind=3), ARG), (dict(ns=0), ARG), (dict(ns=19), ARG),
             (dict(nw2=3), ARG), (dict(s2=0), ARG), (dict(nw2=0), ARG), (dict(ns=1 << 31), ARG),
             (dict(code=L.C64), DT), (dict(code=L.BF16), DT), (dict(code=99), DT)]
    assert_rejected(lambda a: c_radon_patches(pm, *a.values()), base, cases, y)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the operators
# ---------------------------------------------------------------------------------------------------------------
def device_lib(pm):
    return lambda name: getattr(pm.local, name)


def blockdiag(pm, ng, c, dt):
    return pm.MPIBlockDiag([mgp.make(c, dt, device_lib(pm)) for _ in range(ng)], dtype=dt)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_operator_vs_reference_fixtures(pm, case, P):
    """exact cases bit for bit in every dtype, the others in float64 and float32 under a rounding bound of the
    float64 fixture; the P ranks' sections as one rank's blocks"""
    ex = mgp.exact(*case)
    for dt in mgp.DTYPES if ex else ("float64", "float32"):
        x, v = mgp.case_inputs(case, dt)
        Op = blockdiag(pm, sum(rows_of(P, mgp.NG)), case, dt)
        S = Op.ops[0] if hasattr(Op, "ops") else None
        if S is not None:
            assert (S._fused is not None) == (case[0] == "radon")
        got = host((Op @ pm.DistributedArray.to_dist(x)).asarray())
        gota = host((Op.H @ pm.DistributedArray.to_dist(v)).asarray())
        assert got.dtype == np.dtype(dt) and gota.dtype == np.dtype(dt)
        if ex:
            gy, gya = decode(GOLD, mgp.key(*case), dt, mgp.ENC)
            np.testing.assert_array_equal(got, gy)
            np.testing.assert_array_equal(gota, gya)
            continue
        gy, gya = decode(GOLD, mgp.key(*case), "float64", 1)
        if dt == "float64":
            bx, bv = np.abs(x.astype(np.float64)), np.abs(v.astype(np.float64))
        else:
            bx, bv = np.abs(x).astype(np.float64), np.abs(v).astype(np.float64)
        So = mgp.make(case, "float64", mgp.refshim_lib)
        M = np.abs(np.stack([So.matvec(e) for e in np.eye(So.shape[1])], 1))
        nm, nd = mgp.sizes(case)
        k = max(int(np.count_nonzero(M, 1).max()), int(np.count_nonzero(M, 0).max()))
        rdt = np.float32 if dt == "float32" else np.float64
        bnd = np.concatenate([M @ bx[g * nm:(g + 1) * nm] for g in range(mgp.NG)])
        bnda = np.concatenate([M.T @ bv[g * nd:(g + 1) * nd] for g in range(mgp.NG)])
        check_close(got.astype(np.float64), gy, bnd, k, rdt)
        check_close(gota.astype(np.float64), gya, bnda, k, rdt)


def dottest_op(pm, inner):
    rng = np.random.default_rng(9)
    L = pm.local
    if inner == "patch3d":
        t = np.arange(40) * 0.004
        R = L.Radon3D(t, np.arange(6) * 10.0, np.arange(8) * 10.0, np.linspace(-1e-3, 1e-3, 3),
                      np.linspace(-2e-3, 2e-3, 5), kind="parabolic")
        nw, dims, _, _ = L.patch3d_design((15, 20, 100), (6, 8, 40), (3, 4, 20), (3, 5, 40))
        return L.Patch3D(R, dims, (15, 20, 100), (6, 8, 40), (3, 4, 20), (3, 5, 40))
    if inner == "sliding1d":
        M = L.MatrixMult(rng.standard_normal((64, 20)))
        nw, dim, _, _ = L.sliding1d_design(600, 64, 32, 20)
        return L.Sliding1D(M, dim, 600, 64, 32, tapertype="cosine")
    t = np.arange(128) * 0.004
    if inner == "patch2d":
        R = L.Radon2D(t, np.arange(32) * 12.5, np.linspace(0.0, 3000.0, 40), kind="hyperbolic")
        nop = (40, 128)
    else:
        R = L.MatrixMult(rng.standard_normal((32 * 128, 50)))
        nop = (5, 10)
    nw, dims, _, _ = L.patch2d_design((150, 300), (32, 128), (16, 64), nop)
    return L.Patch2D(R, dims, (150, 300), (32, 128), (16, 64), nop, tapertype="cosine")


@pytest.mark.gpu
@pytest.mark.parametrize("inner", ["patch2d", "patch3d", "matrix2d", "sliding1d"])
def test_operator_dottest(pm, inner):
    from pylops_mpi_b200.utils.dottest import dottest
    rng = np.random.default_rng(8)
    S = dottest_op(pm, inner)
    assert (S._fused is not None) == (inner in ("patch2d", "patch3d"))
    Op = pm.MPIBlockDiag([S, S])
    u = pm.DistributedArray.to_dist(rng.standard_normal(Op.shape[1]))
    v = pm.DistributedArray.to_dist(rng.standard_normal(Op.shape[0]))
    assert dottest(Op, u, v, rtol=1e-12)


@pytest.mark.gpu
def test_operator_attributes_and_paths(pm):
    L = pm.local
    t = np.arange(8) * 0.004
    R = L.Radon2D(t, np.arange(8) * 10.0, np.linspace(-1e-3, 1e-3, 4))
    P = L.Patch2D(R, (12, 24), (22, 20), (8, 8), (3, 3), (4, 8), name="W")
    assert (P.dims, P.dimsd, P.shape) == ((12, 24), (22, 20), (440, 288))
    assert (P.nwin, P.nover, P.nop, P.tapertype, P.name, P.dtype, P.scalings) == ((8, 8), (3, 3), (4, 8), "hanning",
                                                                                  "W", np.float64, None)
    assert P._fused is R
    M = L.MatrixMult(np.ones((64, 36), dtype=np.float32))
    P = L.Patch2D(M, (18, 18), (22, 20), (8, 8), (3, 3), (6, 6), tapertype=None)
    assert P._fused is None and P.dtype == np.float32 and P.tapertype is None and P.name == "P"
    R3 = L.Radon3D(t, np.arange(6) * 10.0, np.arange(6) * 10.0, np.linspace(-1e-3, 1e-3, 2),
                   np.linspace(-1e-3, 1e-3, 3))
    P3 = L.Patch3D(R3, (4, 6, 16), (9, 10, 14), (6, 6, 8), (3, 3, 3), (2, 3, 8))
    assert (P3.dims, P3.dimsd, P3.nwin, P3.nover, P3.nop) == ((4, 6, 16), (9, 10, 14), (6, 6, 8), (3, 3, 3),
                                                              (2, 3, 8))
    assert P3._fused is R3
    S = L.Sliding1D(L.MatrixMult(np.ones((8, 3))), 9, 22, 8, 3)
    assert (S.dims, S.dimsd, S.shape, S.nwin, S.nover, S.name) == ((9,), (22,), (22, 9), 8, 3, "S")
    assert S._fused is None
    with pytest.raises(TypeError):
        L.Patch2D(R.H, (12, 24), (22, 20), (8, 8), (3, 3), (4, 8))
    with pytest.raises(TypeError):
        L.Patch2D(R.H @ R, (12, 24), (22, 20), (8, 8), (3, 3), (4, 8))


# the _KernelOperator contract checks of test_local_apply.py, on patch operators
F32R, F64R = ("F32", "F32", "C64", "C128"), ("F64", "F64", "C128", "C128")
CONTRACT = {"Patch2D-Radon2D": ("float64", F64R), "Patch3D-Radon3D": ("float32", F32R),
            "Patch2D-MatrixMult": ("float32", F32R), "Sliding1D-MatrixMult": ("float64", F64R)}


def make_contract(pm, name):
    rng = np.random.default_rng(5)
    L = pm.local
    t = np.arange(6) * 0.004
    dt = CONTRACT[name][0]
    if name == "Patch2D-Radon2D":
        R = L.Radon2D(t, np.arange(6) * 10.0, np.linspace(-1e-3, 1e-3, 3), dtype=dt)
        return L.Patch2D(R, (9, 18), (14, 14), (6, 6), (2, 2), (3, 6))
    if name == "Patch3D-Radon3D":
        R = L.Radon3D(t, np.arange(4) * 10.0, np.arange(4) * 10.0, np.linspace(-1e-3, 1e-3, 2),
                      np.linspace(-1e-3, 1e-3, 2), dtype=dt)
        return L.Patch3D(R, (4, 6, 18), (6, 8, 14), (4, 4, 6), (2, 2, 2), (2, 2, 6))
    if name == "Patch2D-MatrixMult":
        return L.Patch2D(L.MatrixMult(rng.standard_normal((6 * 6, 4)).astype(dt)), (6, 6), (14, 14), (6, 6), (2, 2),
                         (2, 2), tapertype="cosine")
    return L.Sliding1D(L.MatrixMult(rng.standard_normal((6, 4)).astype(dt)), 12, 14, 6, 2)


CHECKS = ["test_result_dtype", "test_out_equals_out_none", "test_complex_data_equals_its_parts",
          "test_complex_into_real_out_warns_and_keeps_the_real_part", "test_wrong_length_raises",
          "test_direct_out_allocates_nothing", "test_graph_safe_by_type"]


@pytest.mark.gpu
@pytest.mark.parametrize("check", CHECKS)
@pytest.mark.parametrize("name", list(CONTRACT))
def test_kernel_operator_contract(pm, monkeypatch, name, check):
    """each check of test_local_apply.py, run on the patch operators through its own registry"""
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
    t = np.arange(32) * 0.004
    if inner == "radon":
        Op1 = L.Radon2D(t, np.arange(12) * 10.0, np.linspace(-1e-3, 1e-3, 21))
        nop = (21, 32)
    else:
        Op1 = L.MatrixMult(rng.standard_normal((12 * 32, 40)))
        nop = (8, 5)
    nw, dims, _, _ = L.patch2d_design((30, 64), (12, 32), (6, 16), nop)
    Op = pm.MPIBlockDiag([L.Patch2D(Op1, dims, (30, 64), (12, 32), (6, 16), nop) for _ in range(2)])
    y = Op @ pm.DistributedArray.to_dist(rng.standard_normal(Op.shape[1]))
    assert_cgls_replay_matches_steps(pm, Op, y, pm.DistributedArray.to_dist(np.zeros(Op.shape[1])), 25, 20)


def flow_tolerance():
    """(x, cost) relative tolerances of the flow, as test_sliding's: 100 times the 4-ulp jitter spread of the
    reference's own run, and no less than 10 cond 2^-53"""
    floor = 10 * float(GOLD["flow/cond"]) * 2.0 ** -53
    return tuple(max(100 * float(s), floor) for s in GOLD["flow/spread"])


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
def test_local_denoising_fista_vs_reference(pm, P):
    alpha = float(GOLD["flow/alpha"])
    Op = pm.MPIBlockDiag([mgp.flow_ops(device_lib(pm)) for r in rows_of(P, mgp.FLOW_NG) for _ in range(r)])
    assert Op.ops[0]._fused is not None
    x0 = pm.DistributedArray.to_dist(np.zeros(Op.shape[1]))
    x, iiter, cost = pm.fista(Op, pm.DistributedArray.to_dist(GOLD["flow/d"]), x0, niter=mgp.FLOW_NITER,
                              eps=mgp.FLOW_EPS, alpha=alpha, tol=1e-10)
    assert iiter == int(GOLD[f"flow/P{P}/iiter"])
    xtol, ctol = flow_tolerance()
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"flow/P{P}/cost"], rtol=ctol)
    gx = GOLD[f"flow/P{P}/x"]
    np.testing.assert_allclose(host(x.asarray()), gx, rtol=0, atol=xtol * np.abs(gx).max())


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [1, 2])
def test_multi_rank_fixtures(nproc):
    needs_gpus(nproc)
    run_on_ranks("test_patch", nproc)


def on_ranks(pm, comm):
    """each rank's MPIBlockDiag of patch operators against its slice of the gathered exact fixtures, and the fista
    flow against its fixture"""
    rank, P = comm.Get_rank(), comm.Get_size()

    def split(n_per, ng):
        rows = rows_of(P, ng)
        lo, hi = sum(rows[:rank]) * n_per, sum(rows[:rank + 1]) * n_per
        return [(r * n_per,) for r in rows], slice(lo, hi), rows[rank]

    for case in mgp.cases():
        if not mgp.exact(*case):
            continue
        nm, nd = mgp.sizes(case)
        lsm, slm, ng = split(nm, mgp.NG)
        lsd, sld, _ = split(nd, mgp.NG)
        for dt in mgp.DTYPES:
            x, v = mgp.case_inputs(case, dt)
            Op = blockdiag(pm, ng, case, dt)
            gy, gya = decode(GOLD, mgp.key(*case), dt, mgp.ENC)
            name = f"{mgp.key(*case)}/{dt}"
            np.testing.assert_array_equal(host((Op @ pm.DistributedArray.to_dist(x, local_shapes=lsm)).local_array),
                                          gy[sld], err_msg=f"[rank {rank}] {name}/y")
            np.testing.assert_array_equal(host((Op.H @ pm.DistributedArray.to_dist(v, local_shapes=lsd)).local_array),
                                          gya[slm], err_msg=f"[rank {rank}] {name}/ya")

    nd = mgp.FLOW_N * mgp.FLOW_NT
    nm = mgp.flow_ops(device_lib(pm)).shape[1]
    lsd, sld, ng = split(nd, mgp.FLOW_NG)
    lsm, slm, _ = split(nm, mgp.FLOW_NG)
    Op = pm.MPIBlockDiag([mgp.flow_ops(device_lib(pm)) for _ in range(ng)])
    d = pm.DistributedArray.to_dist(GOLD["flow/d"], local_shapes=lsd)
    x0 = pm.DistributedArray.to_dist(np.zeros(mgp.FLOW_NG * nm), local_shapes=lsm)
    x, iiter, cost = pm.fista(Op, d, x0, niter=mgp.FLOW_NITER, eps=mgp.FLOW_EPS, alpha=float(GOLD["flow/alpha"]),
                              tol=1e-10)
    assert iiter == int(GOLD[f"flow/P{P}/iiter"])
    xtol, ctol = flow_tolerance()
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"flow/P{P}/cost"], rtol=ctol, err_msg=f"[rank {rank}] cost")
    gx = GOLD[f"flow/P{P}/x"]
    np.testing.assert_allclose(host(x.local_array), gx[slm], rtol=0, atol=xtol * np.abs(gx).max(),
                               err_msg=f"[rank {rank}] x")
