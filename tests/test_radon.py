"""Rank-local Radon2D / Radon3D (pylops.signalprocessing.Radon2D / Radon3D inside MPIBlockDiag, one CMP gather per
block).  On unitless axes, model sample (p, t0) reaches trace h at

    linear      tdec = (t0 + px*hx) + py*hy
    parabolic   tdec = (t0 + px*(hx*hx)) + py*(hy*hy)
    hyperbolic  tdec = sqrt((t0*t0 + (hx/px)*(hx/px)) + (hy/py)*(hy/py))      (2-D: no y term)

in float64; with interp the pair spreads onto it = trunc(tdec), it + 1 with weights 1 - d, d iff 0 <= tdec < nt - 1,
without onto it iff 0 <= tdec < nt; the adjoint is the exact transpose.

CPU: refshim's restatement (tests/golden/refshim/pylops/signalprocessing/radon2d.py, radon3d.py) against a dense
matrix built directly from that definition, argument errors, and the fixtures of tests/golden/radon_golden.npz (made
by make_golden_radon.py: the reference's MPIBlockDiag and FISTA over the restatement).  GPU: the b2_radon kernel
through the C ABI and the operators through the public interface."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_radon as mgr  # noqa: E402
from fixture_codec import decode, rows_of  # noqa: E402
from op_checks import (assert_cgls_replay_matches_steps, assert_rejected, guarded_twice, host,  # noqa: E402
                       needs_gpus, run_on_ranks)

GOLD = np.load(os.path.join(HERE, "golden", "radon_golden.npz"), allow_pickle=False)
CASES = mgr.cases()
KINDS = mgr.KINDS
U64, U32 = 2.0 ** -53, 2.0 ** -24


# ---------------------------------------------------------------------------------------------------------------
# the definition, built directly
# ---------------------------------------------------------------------------------------------------------------
def tdec(kind, t0, hx, px, hy=None, py=None):
    """tdec of the model samples t0 (an int array) for one pair of traces, NumPy float64 operations in the pinned
    order (elementwise IEEE operations: no contraction)"""
    t0 = np.asarray(t0, dtype=np.int64)
    hx, px = np.float64(hx), np.float64(px)
    with np.errstate(divide="ignore", invalid="ignore"):
        if kind == "hyperbolic":
            q = hx / px
            v = (t0 * t0).astype(np.float64) + q * q
            if hy is not None:
                r = np.float64(hy) / np.float64(py)
                v = v + r * r
            return np.sqrt(v)
        cx = px * hx if kind == "linear" else px * (hx * hx)
        v = t0.astype(np.float64) + cx
        if hy is not None:
            hy, py = np.float64(hy), np.float64(py)
            v = v + (py * hy if kind == "linear" else py * (hy * hy))
        return v


def dense(kind, interp, nt, hx, px, hy=None, py=None):
    """the operator's matrix, data (hy, hx, t) x model (py, px, t0), from unitless axes (hy = py = None: 2-D)"""
    nhy = 1 if hy is None else len(hy)
    npy = 1 if py is None else len(py)
    M = np.zeros((nhy * len(hx) * nt, npy * len(px) * nt))
    t0 = np.arange(nt)
    for jy in range(nhy):
        for jx, h in enumerate(hx):
            for iy in range(npy):
                for ix, p in enumerate(px):
                    v = tdec(kind, t0, h, p, None if hy is None else hy[jy], None if py is None else py[iy])
                    ok = (v >= 0) & (v < (nt - 1 if interp else nt))
                    col = (iy * len(px) + ix) * nt + t0[ok]
                    row = (jy * len(hx) + jx) * nt
                    it = np.floor(v[ok]).astype(np.int64)
                    if interp:
                        d = v[ok] - it
                        M[row + it, col] += 1 - d
                        M[row + it + 1, col] += d
                    else:
                        M[row + it, col] += 1
    return M


def unitless(kind, dt, haxis, paxis, centeredh):
    """the axes as the operators make them unitless (the pinned host conventions)"""
    haxis, paxis = np.asarray(haxis, dtype=np.float64), np.asarray(paxis, dtype=np.float64)
    dh = abs(haxis[1] - haxis[0])
    nh = haxis.size
    h = np.arange(nh) - nh // 2 + ((nh + 1) % 2) / 2 if centeredh else haxis / dh
    return h, paxis * {"linear": dh / dt, "parabolic": dh * dh / dt, "hyperbolic": dt / dh}[kind]


def restated(ndim):
    return mgr.restated(ndim)


def random_geometry(rng, kind, ndim):
    """physical axes with irregular values (not dyadic), a zero velocity for hyperbolic"""
    dt = 0.004
    t = np.arange(23) * dt
    hs = [np.arange(n) * dh + o for n, dh, o in ((5, 12.5, -20.0), (6, 10.0, 3.0))[3 - ndim:]]
    scale = {"linear": 1e-3, "parabolic": 1e-5, "hyperbolic": 2e3}[kind]
    ps = [rng.uniform(-1, 1, n) * scale for n in (3, 4)[3 - ndim:]]
    if kind == "hyperbolic":
        ps = [np.abs(p) for p in ps]
        ps[-1][0] = 0.0
    return t, hs, ps


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("centeredh", [True, False], ids=["centred", "haxis"])
@pytest.mark.parametrize("interp", [True, False], ids=["interp", "nointerp"])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("ndim", [2, 3], ids=["2d", "3d"])
def test_restatement_is_the_dense_definition(ndim, kind, interp, centeredh):
    rng = np.random.default_rng(3 * ndim + KINDS.index(kind))
    t, hs, ps = random_geometry(rng, kind, ndim)
    R = restated(ndim)(t, *hs, *ps, kind=kind, centeredh=centeredh, interp=interp)
    ax = [unitless(kind, 0.004, h, p, centeredh) for h, p in zip(hs, ps)]
    if ndim == 2:
        M = dense(kind, interp, t.size, ax[0][0], ax[0][1])
    else:
        M = dense(kind, interp, t.size, ax[1][0], ax[1][1], ax[0][0], ax[0][1])
    assert R.shape == M.shape and np.count_nonzero(M) > 0
    np.testing.assert_array_equal(mgr.dense(R), M)
    Ma = np.stack([R.rmatvec(e) for e in np.eye(M.shape[0])], 1)
    np.testing.assert_array_equal(Ma, M.T)


def test_restatement_argument_errors():
    R2, R3 = restated(2), restated(3)
    t, h, p = np.arange(8) * 0.004, np.arange(4) * 10.0, np.linspace(-1e-3, 1e-3, 3)
    with pytest.raises(NotImplementedError, match="kind"):
        R2(t, h, p, kind="cubic")
    with pytest.raises(NotImplementedError, match="dtype"):
        R2(t, h, p, dtype="complex128")
    with pytest.raises(KeyError):
        R2(t, h, p, engine="torch")
    for bad in ((t[:1], h, p), (t, h[:1], p)):
        with pytest.raises(ValueError):
            R2(*bad)
    with pytest.raises(ValueError):
        R3(t, h[:1], h, p, p)


def test_operator_argument_errors_before_any_device_work():
    import pylops_mpi_b200 as pm
    t, h, p = np.arange(8) * 0.004, np.arange(4) * 10.0, np.linspace(-1e-3, 1e-3, 3)
    with pytest.raises(NotImplementedError, match="kind"):
        pm.local.Radon2D(t, h, p, kind="cubic")
    for dt in ("complex128", "complex64"):
        with pytest.raises(NotImplementedError, match="dtype"):
            pm.local.Radon2D(t, h, p, dtype=dt)
    with pytest.raises(KeyError):
        pm.local.Radon2D(t, h, p, engine="torch")
    with pytest.raises(ValueError):
        pm.local.Radon2D(t[:1], h, p)
    with pytest.raises(ValueError):
        pm.local.Radon2D(t, h[:1], p)
    with pytest.raises(ValueError):
        pm.local.Radon3D(t, h, h[:1], p, p)


def case_id(c):
    return mgr.key(*c)[3:]


def test_fixture_inventory():
    want = set()
    for c in CASES:
        k = mgr.key(*c)
        nm, nd = mgr.sizes(c[0], c[1], c[4])
        ex = mgr.exact(c[1], c[2])
        names = ("y", "ya", "yi", "yai") if mgr.complex_case(*c[1:4]) else ("y", "ya")
        for n in names:
            a = GOLD[f"{k}/{n}"]
            assert a.dtype == (np.int32 if ex or n in ("yi", "yai") else np.float64)
            assert a.shape == (mgr.NG * (nd if n in ("y", "yi") else nm),)
            want.add(f"{k}/{n}")
    assert len(CASES) == 3 * 2 * 2 * 3
    want |= {"flow/d", "flow/m", "flow/alpha", "flow/cond", "flow/spread"}
    want |= {f"flow/P{P}/{k}" for P in (1, 2, 3) for k in ("x", "iiter", "cost")}
    assert sorted(GOLD.files) == sorted(want)
    assert GOLD["flow/spread"].shape == (2,) and float(GOLD["flow/spread"].max()) < 1e-10
    for P in (1, 2, 3):
        assert int(GOLD[f"flow/P{P}/iiter"]) == mgr.FLOW_NITER
        assert GOLD[f"flow/P{P}/cost"].shape == (mgr.FLOW_NITER,)


def restated_gathers(c, dt):
    """forward of x and adjoint of v, gather by gather, through the restatement (dtype dt of the data)"""
    ndim, kind, interp, centeredh, nh = c
    x, v = mgr.case_inputs(*c, dt)
    nm, nd = mgr.sizes(ndim, kind, nh)
    R = restated(ndim)(mgr.taxis(ndim), *mgr.axes(ndim, kind, centeredh, nh), kind=kind, centeredh=centeredh,
                       interp=interp, dtype="float32" if dt == "float32" else "float64")
    y = np.concatenate([R.matvec(x[g * nm:(g + 1) * nm]) for g in range(mgr.NG)])
    ya = np.concatenate([R.rmatvec(v[g * nd:(g + 1) * nd]) for g in range(mgr.NG)])
    return y, ya


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_fixtures_follow_the_restatement_in_every_dtype(case):
    ex = mgr.exact(case[1], case[2])
    for dt in mgr.DTYPES:
        if dt == "complex128" and not mgr.complex_case(*case[1:4]):
            continue
        y, ya = restated_gathers(case, dt)
        gy, gya = decode(GOLD, mgr.key(*case), dt, mgr.ENC if ex else 1)
        assert y.dtype == np.dtype(dt)
        np.testing.assert_array_equal(y, gy)
        np.testing.assert_array_equal(ya, gya)


def test_flow_inputs_regenerate():
    m, d, alpha = mgr.flow_inputs()
    np.testing.assert_array_equal(m.ravel(), GOLD["flow/m"])
    np.testing.assert_array_equal(d, GOLD["flow/d"])
    assert alpha == float(GOLD["flow/alpha"])


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernel through the C ABI
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


def c_radon(pm, x, y, nt, n_inner, ny, nx, my, mx, hy, hx, py, px, kind, interp, adjoint, code):
    L = pm._lib
    return L.lib.b2_radon(L.ctx(), x, y, nt, n_inner, ny, nx, my, mx, hy, hx, py, px, kind, interp, adjoint, code,
                          L.stream())


def run_kernel(pm, x_np, nt, hx, px, hy, py, kind, interp, adjoint, dt, guard=3):
    """apply through the C ABI into a guarded view; x_np float64 / complex128 values representable in dt.
    Returns (y as float64 / complex128, guards intact, second apply bit-equal)"""
    import torch
    cplx = np.iscomplexobj(x_np)
    xr = np.stack([x_np.real, x_np.imag], -1).ravel() if cplx else x_np.ravel()
    C = 2 if cplx else 1
    dev = [None if a is None else torch.as_tensor(np.asarray(a, dtype=np.float64)).cuda() for a in (hy, hx, py, px)]
    ptrs = [0 if a is None else a.data_ptr() for a in dev]
    nhy, npy = (1 if hy is None else len(hy)), (1 if py is None else len(py))
    nout = (npy * len(px) if adjoint else nhy * len(hx)) * nt * C
    x = torch.as_tensor(xr.astype(dt)).cuda()
    code = pm._lib.F32 if dt == np.float32 else pm._lib.F64
    args = (nt, C, nhy, len(hx), npy, len(px), ptrs[0] or None, ptrs[1], ptrs[2] or None, ptrs[3],
            mgr.KINDS.index(kind), int(interp), int(adjoint), code)
    first, guards, same = guarded_twice(lambda yp: c_radon(pm, x.data_ptr(), yp, *args), nout, dt, guard)
    out = first.astype(np.float64)
    if cplx:
        out = out[0::2] + 1j * out[1::2]
    return out, guards, same


def check_close(got, A, x, dt):
    """got ~ A x componentwise: a float64 sum of k terms is within (k + 2) u of sum |terms|, and float32 results are
    rounded once more"""
    ref = A @ x
    bnd = np.abs(A) @ np.abs(x)
    k = max(int(np.count_nonzero(A, 1).max()), 1)
    tol = (k + 2) * U64 * bnd + (U32 * np.abs(ref) if dt == np.float32 else 0)
    err = np.abs(got - ref)
    assert np.all(err <= tol + 1e-300), f"max err {err.max():.3e}, worst ratio {np.max(err / (tol + 1e-300)):.3f}"


def kernel_axes(kind, ndim, rng, nhs=(3, 5), nps=(2, 4)):
    """unitless axes (hy, hx, py, px) with irregular values, a zero velocity for hyperbolic (2-D: hy = py = None)"""
    hx = np.sort(rng.uniform(-8, 8, nhs[1]))
    px = rng.uniform(-1.5, 1.5, nps[1]) if kind == "linear" else (
        rng.uniform(-0.2, 0.2, nps[1]) if kind == "parabolic" else np.abs(rng.uniform(0, 2, nps[1])))
    if kind == "hyperbolic":
        px[0] = 0.0
    if ndim == 2:
        return None, hx, None, px
    hy = np.sort(rng.uniform(-6, 6, nhs[0]))
    py = rng.uniform(-1, 1, nps[0]) * (0.2 if kind == "parabolic" else 1.0)
    if kind == "hyperbolic":
        py = np.abs(py) + 0.5
    return hy, hx, py, px


# (nt, (nhy, nhx), (npy, npx)): more traces and model traces than one 256-term tile, singletons, nt = 2, several
# 256-sample CTAs per trace
KERNEL_SHAPES = [(45, (3, 5), (2, 4)), (3, (2, 300), (1, 270)), (2, (1, 1), (1, 1)), (37, (1, 7), (3, 1)),
                 (600, (1, 2), (2, 1))]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("interp", [True, False], ids=["interp", "nointerp"])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("ndim", [2, 3], ids=["2d", "3d"])
def test_kernel_vs_dense_matrix(pm, ndim, kind, interp, dt):
    rng = np.random.default_rng(10 * ndim + KINDS.index(kind) + 4 * int(interp))
    for nt, nhs, nps in KERNEL_SHAPES:
        hy, hx, py, px = kernel_axes(kind, ndim, rng, nhs, nps)
        M = dense(kind, interp, nt, hx, px, hy, py)
        for cplx in (False, True):
            for adjoint in (False, True):
                n = M.shape[0] if adjoint else M.shape[1]
                x = rng.standard_normal(n).astype(dt).astype(np.float64)
                if cplx:
                    x = x + 1j * rng.standard_normal(n).astype(dt).astype(np.float64)
                y, guards, same = run_kernel(pm, x, nt, hx, px, hy, py, kind, interp, adjoint, dt)
                assert guards and same, (nt, nhs, nps, cplx, adjoint)
                check_close(y, M.T if adjoint else M, x, dt)


@pytest.mark.gpu
def test_kernel_2d_equals_3d_with_singleton_y(pm):
    """a singleton y axis of finite terms (h = 0, p = 1) adds exact zeros: the 3-D path equals the 2-D one bit for
    bit (the 2-D call forms no y term at all, which a hyperbolic 0/0 would need)"""
    rng = np.random.default_rng(4)
    for kind in ("linear", "parabolic"):
        _, hx, _, px = kernel_axes(kind, 2, rng, (1, 40), (1, 33))
        for adjoint in (False, True):
            n = (len(hx) if adjoint else len(px)) * 77
            x = rng.standard_normal(n)
            a = run_kernel(pm, x, 77, hx, px, None, None, kind, True, adjoint, np.float64)[0]
            b = run_kernel(pm, x, 77, hx, px, [0.0], [1.0], kind, True, adjoint, np.float64)[0]
            np.testing.assert_array_equal(a, b)


@pytest.mark.gpu
def test_kernel_error_codes_leave_y_untouched(pm):
    import torch
    L = pm._lib
    ARG, DT = 2002, 2001
    nt, nh, npp = 10, 3, 4
    x = torch.ones(npp * nt, dtype=torch.float64, device="cuda")
    y = torch.full((nh * nt,), 3.5, dtype=torch.float64, device="cuda")
    ax = torch.arange(4, dtype=torch.float64, device="cuda")
    base = dict(x=x.data_ptr(), y=y.data_ptr(), nt=nt, n_inner=1, ny=1, nx=nh, my=1, mx=npp, hy=None,
                hx=ax.data_ptr(), py=None, px=ax.data_ptr(), kind=0, interp=1, adjoint=0, code=L.F64)
    big = 1 << 31
    cases = [
        (dict(x=None), ARG), (dict(y=None), ARG), (dict(y=x.data_ptr()), ARG), (dict(hx=None), ARG),
        (dict(px=None), ARG), (dict(hy=ax.data_ptr()), ARG), (dict(py=ax.data_ptr()), ARG),
        (dict(ny=2), ARG), (dict(my=2), ARG),
        (dict(nt=0), ARG), (dict(nx=0), ARG), (dict(mx=0), ARG), (dict(nt=big), ARG), (dict(nx=big), ARG),
        (dict(mx=big), ARG), (dict(hy=ax.data_ptr(), py=ax.data_ptr(), ny=big), ARG),
        (dict(hy=ax.data_ptr(), py=ax.data_ptr(), my=0), ARG),
        (dict(n_inner=0), ARG), (dict(n_inner=3), ARG), (dict(kind=3), ARG), (dict(kind=-1), ARG),
        (dict(nt=1 << 30, nx=1 << 20), ARG),                                     # more CTAs than one grid holds
        (dict(code=L.C64), DT), (dict(code=L.C128), DT), (dict(code=L.BF16), DT), (dict(code=99), DT),
    ]
    assert_rejected(lambda a: c_radon(pm, *a.values()), base, cases, y)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the operators
# ---------------------------------------------------------------------------------------------------------------
def blockdiag(pm, P, case, dt):
    """P ranks' gathers as one rank's blocks (the gathered result does not depend on how they are split)"""
    ndim, kind, interp, centeredh, nh = case
    cls = pm.local.Radon2D if ndim == 2 else pm.local.Radon3D
    ops = [cls(mgr.taxis(ndim), *mgr.axes(ndim, kind, centeredh, nh), kind=kind, centeredh=centeredh, interp=interp,
               dtype="float32" if dt == "float32" else "float64") for r in rows_of(P, mgr.NG) for _ in range(r)]
    return pm.MPIBlockDiag(ops, dtype=dt)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_operator_vs_reference_fixtures(pm, case, P):
    """exact cases bit for bit in every dtype; hyperbolic curves with interpolation under the rounding bound of the
    gather-by-gather dense matrix"""
    ex = mgr.exact(case[1], case[2])
    for dt in mgr.DTYPES:
        if dt == "complex128" and not mgr.complex_case(*case[1:4]):
            continue
        x, v = mgr.case_inputs(*case, dt)
        Op = blockdiag(pm, P, case, dt)
        got = host((Op @ pm.DistributedArray.to_dist(x)).asarray())
        gota = host((Op.H @ pm.DistributedArray.to_dist(v)).asarray())
        assert got.dtype == np.dtype(dt) and gota.dtype == np.dtype(dt)
        gy, gya = decode(GOLD, mgr.key(*case), dt, mgr.ENC if ex else 1)
        if ex:
            np.testing.assert_array_equal(got, gy)
            np.testing.assert_array_equal(gota, gya)
            continue
        ndim, kind, interp, centeredh, nh = case
        R = restated(ndim)(mgr.taxis(ndim), *mgr.axes(ndim, kind, centeredh, nh), kind=kind, centeredh=centeredh,
                           interp=interp)
        M = mgr.dense(R)
        nm, nd = mgr.sizes(ndim, kind, nh)
        rdt = np.float32 if dt == "float32" else np.float64
        for g in range(mgr.NG):
            check_close(got[g * nd:(g + 1) * nd].astype(np.float64), M, x[g * nm:(g + 1) * nm].astype(np.float64), rdt)
            check_close(gota[g * nm:(g + 1) * nm].astype(np.float64), M.T, v[g * nd:(g + 1) * nd].astype(np.float64),
                        rdt)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_operator_dottest_multi_tile(pm, kind):
    from pylops_mpi_b200.utils.dottest import dottest
    rng = np.random.default_rng(8)
    t = np.arange(700) * 0.002
    h = np.arange(300) * 12.5
    p = {"linear": np.linspace(-4e-4, 4e-4, 300), "parabolic": np.linspace(-2e-7, 2e-7, 300),
         "hyperbolic": np.linspace(0.0, 4000.0, 300)}[kind]
    Op = pm.MPIBlockDiag([pm.local.Radon2D(t, h, p, kind=kind), pm.local.Radon2D(t, h, p, kind=kind, centeredh=False)])
    u = pm.DistributedArray.to_dist(rng.standard_normal(Op.shape[1]))
    v = pm.DistributedArray.to_dist(rng.standard_normal(Op.shape[0]))
    assert dottest(Op, u, v, rtol=1e-12)


@pytest.mark.gpu
def test_operator_attributes_dtypes_and_out(pm):
    import torch
    t, hy, hx = np.arange(50) * 0.004, np.arange(3) * 20.0, np.arange(5) * 10.0
    py, px = np.linspace(-1e-3, 1e-3, 2), np.linspace(-2e-3, 2e-3, 4)
    R2 = pm.local.Radon2D(t, hx, px, kind="parabolic", interp=False, name="Q")
    assert R2.dims == (4, 50) and R2.dimsd == (5, 50) and R2.shape == (250, 200)
    assert (R2.kind, R2.interp, R2.engine, R2.name, R2.dtype) == ("parabolic", False, "numpy", "Q", np.float64)
    R3 = pm.local.Radon3D(t, hy, hx, py, px, dtype="float32")
    assert R3.dims == (2, 4, 50) and R3.dimsd == (3, 5, 50) and R3.shape == (750, 400)
    assert (R3.kind, R3.interp, R3.name, R3.dtype) == ("linear", True, "R", np.float32)
    rng = np.random.default_rng(2)
    for R in (R2, R3):
        same = [type(R)(t, *((hy, hx, py, px) if R is R3 else (hx, px)), kind=R.kind, interp=R.interp, dtype=R.dtype,
                        onthefly=True, engine=e) for e in ("numpy", "numba", "cuda")]
        x = torch.as_tensor(rng.standard_normal(R.shape[1])).cuda()
        v = torch.as_tensor(rng.standard_normal(R.shape[0])).cuda()
        ref, refa = R.matvec(x), R.rmatvec(v)
        for S in same:
            assert torch.equal(S.matvec(x), ref) and torch.equal(S.rmatvec(v), refa)
        assert torch.equal(R.H.matvec(v), refa)
    # dtype promotion: the float32 operator computes float64-typed complex data in complex128
    z = torch.complex(torch.ones(400, dtype=torch.float64), torch.ones(400, dtype=torch.float64)).cuda()
    assert R3.matvec(z).dtype == torch.complex128


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_cgls_graph_replay_matches_step_loop(pm, kind):
    rng = np.random.default_rng(12)
    t, h = np.arange(96) * 0.004, np.arange(24) * 10.0
    p = {"linear": np.linspace(-1e-3, 1e-3, 31), "parabolic": np.linspace(-5e-6, 5e-6, 31),
         "hyperbolic": np.linspace(1500.0, 4000.0, 31)}[kind]
    Op = pm.MPIBlockDiag([pm.local.Radon2D(t, h, p, kind=kind) for _ in range(3)])
    y = Op @ pm.DistributedArray.to_dist(rng.standard_normal(Op.shape[1]))
    assert_cgls_replay_matches_steps(pm, Op, y, pm.DistributedArray.to_dist(np.zeros(Op.shape[1])), 25, 20)


def flow_tolerance():
    """(x, cost) relative tolerances of the flow: a run summed in another order than the restatement moves by about
    what a 4-ulp jitter of every apply moves the reference's own run (``spread``), and by no less than cond * 2^-53;
    the test allows 100 and 10 times those"""
    floor = 10 * float(GOLD["flow/cond"]) * 2.0 ** -53
    return tuple(max(100 * float(s), floor) for s in GOLD["flow/spread"])


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
def test_denoising_fista_vs_reference(pm, P):
    t, h, p = mgr.flow_axes()
    alpha = float(GOLD["flow/alpha"])
    d = GOLD["flow/d"]
    Op = pm.MPIBlockDiag([pm.local.Radon2D(t, h, p, kind="linear") for r in rows_of(P, mgr.FLOW_NG)
                          for _ in range(r)])
    x0 = pm.DistributedArray.to_dist(np.zeros(Op.shape[1]))
    x, iiter, cost = pm.fista(Op, pm.DistributedArray.to_dist(d), x0, niter=mgr.FLOW_NITER, eps=mgr.FLOW_EPS,
                              alpha=alpha, tol=1e-10)
    assert iiter == int(GOLD[f"flow/P{P}/iiter"])
    xtol, ctol = flow_tolerance()
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"flow/P{P}/cost"], rtol=ctol)
    gx = GOLD[f"flow/P{P}/x"]
    np.testing.assert_allclose(host(x.asarray()), gx, rtol=0, atol=xtol * np.abs(gx).max())


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [1, 2])
def test_multi_rank_fixtures(nproc):
    needs_gpus(nproc)
    run_on_ranks("test_radon", nproc)


def on_ranks(pm, comm):
    """each rank's MPIBlockDiag of Radon2D / Radon3D against its slice of the gathered fixtures, and the fista
    denoising flow against its fixture"""
    rank, P = comm.Get_rank(), comm.Get_size()

    def split(n_per, ng=mgr.NG):
        """local shapes of ng gathers of n_per values over the ranks, and this rank's slice"""
        rows = rows_of(P, ng)
        lo, hi = sum(rows[:rank]) * n_per, sum(rows[:rank + 1]) * n_per
        return [(r * n_per,) for r in rows], slice(lo, hi), rows[rank]

    for case in mgr.cases():
        ndim, kind, interp, centeredh, nh = case
        if not mgr.exact(kind, interp):
            continue
        nm, nd = mgr.sizes(ndim, kind, nh)
        lsm, slm, ng = split(nm)
        lsd, sld, _ = split(nd)
        cls = pm.local.Radon2D if ndim == 2 else pm.local.Radon3D
        for dt in mgr.DTYPES:
            if dt == "complex128" and not mgr.complex_case(kind, interp, centeredh):
                continue
            x, v = mgr.case_inputs(*case, dt)
            Op = pm.MPIBlockDiag([cls(mgr.taxis(ndim), *mgr.axes(ndim, kind, centeredh, nh), kind=kind,
                                      centeredh=centeredh, interp=interp, dtype="float32" if dt == "float32" else "float64")
                                  for _ in range(ng)], dtype=dt)
            gy, gya = decode(GOLD, mgr.key(*case), dt, mgr.ENC)
            name = f"{mgr.key(*case)}/{dt}"
            np.testing.assert_array_equal(host((Op @ pm.DistributedArray.to_dist(x, local_shapes=lsm)).local_array),
                                          gy[sld], err_msg=f"[rank {rank}] {name}/y")
            np.testing.assert_array_equal(host((Op.H @ pm.DistributedArray.to_dist(v, local_shapes=lsd)).local_array),
                                          gya[slm], err_msg=f"[rank {rank}] {name}/ya")

    t, h, p = mgr.flow_axes()
    nd, nm = mgr.FLOW_NH * mgr.FLOW_NT, p.size * mgr.FLOW_NT
    lsd, sld, ng = split(nd, mgr.FLOW_NG)
    lsm, slm, _ = split(nm, mgr.FLOW_NG)
    Op = pm.MPIBlockDiag([pm.local.Radon2D(t, h, p, kind="linear") for _ in range(ng)])
    d = pm.DistributedArray.to_dist(GOLD["flow/d"], local_shapes=lsd)
    x0 = pm.DistributedArray.to_dist(np.zeros(mgr.FLOW_NG * nm), local_shapes=lsm)
    x, iiter, cost = pm.fista(Op, d, x0, niter=mgr.FLOW_NITER, eps=mgr.FLOW_EPS, alpha=float(GOLD["flow/alpha"]), tol=1e-10)
    assert iiter == int(GOLD[f"flow/P{P}/iiter"])
    xtol, ctol = flow_tolerance()
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"flow/P{P}/cost"], rtol=ctol, err_msg=f"[rank {rank}] cost")
    gx = GOLD[f"flow/P{P}/x"]
    np.testing.assert_allclose(host(x.local_array), gx[slm], rtol=0, atol=xtol * np.abs(gx).max(),
                               err_msg=f"[rank {rank}] x")
