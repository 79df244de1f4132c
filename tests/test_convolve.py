"""Rank-local Convolve1D (pylops.signalprocessing.Convolve1D inside MPIBlockDiag, tutorials/reflectivity.py:74-76).

    forward  y[i] = sum_k h[k] x[i + offset - k] == np.convolve(x, h, "full")[offset:offset + n]
    adjoint  the exact transpose

CPU: refshim's restatement of pylops 2.x against that definition, and the fixtures of
tests/golden/convolve_golden.npz (made by make_golden_convolve.py: the reference's MPIBlockDiag and ISTA over the
restatement; inputs exactly representable, so every dtype must match them bit for bit).  GPU: the b2_convolve_axis kernel through the C ABI and the operator through the public interface."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_convolve as mgc  # noqa: E402
from fixture_codec import decode, rows_of  # noqa: E402
from op_checks import (assert_cgls_replay_matches_steps, assert_rejected, device_input, guarded_twice, host,  # noqa: E402
                       needs_gpus, run_on_ranks)

GOLD = np.load(os.path.join(HERE, "golden", "convolve_golden.npz"), allow_pickle=False)
CASES = mgc.cases()
U32 = 2.0 ** -24


def conv_ref(x, h, off, adjoint=False, axis=-1):
    """the pinned definition along ``axis`` (float64 / complex128 in NumPy)"""
    h = np.asarray(h, dtype=np.float64)
    nh = h.size
    if adjoint:
        h, off = h[::-1], nh - 1 - off
    x = np.moveaxis(np.asarray(x), axis, -1)
    n = x.shape[-1]
    y = np.zeros(x.shape, dtype=np.result_type(x.dtype, np.float64))
    for k in range(nh):
        s = off - k                        # y[i] += h[k] x[i + s]
        lo, hi = max(0, -s), min(n, n - s)
        if hi > lo:
            y[..., lo:hi] += h[k] * x[..., lo + s:hi + s]
    return np.moveaxis(y, -1, axis)


def bound(x, h, off, adjoint, axis=-1):
    return conv_ref(np.abs(x), np.abs(h), off, adjoint, axis)


def refshim_convolve():
    sys.path.insert(0, os.path.join(HERE, "golden", "refshim"))
    try:
        from pylops.signalprocessing.convolve1d import Convolve1D
    finally:
        sys.path.remove(os.path.join(HERE, "golden", "refshim"))
    return Convolve1D


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nh", range(1, 13))
def test_refshim_restatement_is_the_pinned_definition(nh):
    Convolve1D = refshim_convolve()
    rng = np.random.default_rng(nh)
    h = rng.standard_normal(nh)
    for off in range(nh):
        for n in (1, 3, 30):
            Cop = Convolve1D((n,), h, offset=off)
            eye = np.eye(n)
            M = np.stack([Cop.matvec(e) for e in eye], 1)
            Ma = np.stack([Cop.rmatvec(e) for e in eye], 1)
            Mr = np.stack([np.convolve(e, h, "full")[off:off + n] for e in eye], 1)
            np.testing.assert_allclose(M, Mr, rtol=0, atol=1e-13, err_msg=f"nh={nh} off={off} n={n}")
            np.testing.assert_allclose(Ma, Mr.T, rtol=0, atol=1e-13, err_msg=f"nh={nh} off={off} n={n}")
            np.testing.assert_allclose(conv_ref(eye, h, off), Mr.T, rtol=0, atol=1e-13)


def case_id(c):
    return f"P{c[0]}/ax{c[1]}/nh{c[2]}/o{c[3]}/{c[4]}"


def test_convolve_fixture_inventory():
    assert len(CASES) == 3 * 3 * 10 * 2 + 3 * 3 * 2
    stored = set()
    for P, axis, nh, off, dt in CASES:
        k = mgc.key(P, axis, nh, off)
        for n in ("y", "ya", "yi", "yai")[:4 if dt == "complex128" else 2]:
            a = GOLD[f"{k}/{n}"]
            assert a.dtype == np.int8 and a.shape == (int(np.prod(mgc.DIMS)),)
            stored.add(f"{k}/{n}")
    # axis 0: one entry per P; axes -1 and 1 do not depend on P and are stored once; complex cases add yi, yai
    assert len(stored) == 2 * (3 * 10 + 2 * 10) + 2 * (3 * 2 + 2 * 2)
    for P in (1, 2, 3):
        assert int(GOLD[f"refl/P{P}/iiter"]) == mgc.REFL_NITER
        assert GOLD[f"refl/P{P}/cost"].shape == (mgc.REFL_NITER,)
        assert GOLD[f"refl/P{P}/x"].shape == (int(np.prod(mgc.REFL_DIMS)),)
    assert sorted(GOLD.files) == sorted(stored | {"refl/d", "refl/alpha"} |
                                        {f"refl/P{P}/{k}" for P in (1, 2, 3) for k in ("x", "iiter", "cost")})


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_fixtures_follow_the_pinned_definition(case):
    P, axis, nh, off, dt = case
    h, x, y = mgc.case_inputs(nh, dt)
    parts = np.cumsum([0] + rows_of(P, mgc.DIMS[0]))
    x3, y3 = x.reshape(mgc.DIMS), y.reshape(mgc.DIMS)
    fwd = np.concatenate([conv_ref(x3[a:b], h, off, False, axis) for a, b in zip(parts[:-1], parts[1:])])
    adj = np.concatenate([conv_ref(y3[a:b], h, off, True, axis) for a, b in zip(parts[:-1], parts[1:])])
    gy, gya = decode(GOLD, mgc.key(P, axis, nh, off), dt, mgc.ENC)
    np.testing.assert_array_equal(gy, fwd.ravel())       # exact: every value is a multiple of 1/2
    np.testing.assert_array_equal(gya, adj.ravel())


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernel through the C ABI
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


def c_conv(pm, x, y, shape, h, nh, off, adjoint, dtype_code):
    lib, L = pm._lib.lib, pm._lib
    return lib.b2_convolve_axis(L.ctx(), x, y, shape[0], shape[1], shape[2], h, nh, off, adjoint, dtype_code,
                                L.stream())


NHS = (1, 2, 5, 8, 41, 127, 300)


def axis_lengths(nh):
    return sorted({1, max(1, nh - 1), 37, 4100})


def run_kernel(pm, x_np, h_np, off, adjoint, dt, misalign=False, guard=5):
    """apply through the C ABI into a guarded interior view; returns (y, guards intact, second apply bit-equal)"""
    x, h = device_input(x_np, dt, misalign), device_input(h_np, dt)
    code = pm._lib.F32 if dt == np.float32 else pm._lib.F64
    y, guards_ok, same = guarded_twice(
        lambda yp: c_conv(pm, x.data_ptr(), yp, x_np.shape, h.data_ptr(), h.numel(), off, int(adjoint), code),
        x_np.size, dt, guard, int(misalign))
    return y.reshape(x_np.shape), guards_ok, same


def check_close(got, x, h, off, adjoint, dt, axis=1):
    ref = conv_ref(x.astype(np.float64), h.astype(np.float64), off, adjoint, axis)
    bnd = bound(x.astype(np.float64), h.astype(np.float64), off, adjoint, axis)
    nh = h.size
    tol = (1e-12 * bnd) if dt == np.float64 else (4 * (nh + 2) * U32 * bnd)
    err = np.abs(got.astype(np.float64) - ref)
    assert np.all(err <= tol + 1e-300), f"max err {err.max():.3e}, worst ratio {np.max(err / (tol + 1e-300)):.3f}"


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("n_inner", [1, 3, 8], ids=["inner1", "inner3", "inner8"])
@pytest.mark.parametrize("nh", NHS)
def test_kernel_vs_numpy(pm, dt, n_inner, nh):
    rng = np.random.default_rng(nh * 10 + n_inner)
    h = rng.standard_normal(nh).astype(dt)
    for n in axis_lengths(nh):
        n_outer = 3 if n * n_inner < 20000 else 1
        x = rng.standard_normal((n_outer, n, n_inner)).astype(dt)
        for off in sorted({0, nh // 2, nh - 1}):
            for adjoint in (False, True):
                for misalign in (False, True):
                    y, guards, same = run_kernel(pm, x, h, off, adjoint, dt, misalign)
                    assert guards, (n, off, adjoint, misalign)
                    assert same, (n, off, adjoint, misalign)
                    check_close(y, x, h, off, adjoint, dt)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("n_inner", [1, 4])
def test_kernel_n_outer_beyond_grid_limit(pm, dt, n_inner):
    rng = np.random.default_rng(5)
    h = rng.standard_normal(7).astype(dt)
    x = rng.standard_normal((70001, 5, n_inner)).astype(dt)
    for adjoint in (False, True):
        y, guards, same = run_kernel(pm, x, h, 2, adjoint, dt)
        assert guards and same
        check_close(y, x, h, 2, adjoint, dt)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(4, 300, 1), (3, 50, 6), (2, 7, 16)])
@pytest.mark.parametrize("nh,off", [(5, 1), (41, 20), (130, 3)])
def test_kernel_adjoint_dot(pm, shape, nh, off):
    rng = np.random.default_rng(11)
    h = rng.standard_normal(nh)
    x, v = rng.standard_normal(shape), rng.standard_normal(shape)
    cx, _, _ = run_kernel(pm, x, h, off, False, np.float64)
    chv, _, _ = run_kernel(pm, v, h, off, True, np.float64)
    lhs, rhs = np.vdot(cx, v), np.vdot(x, chv)
    assert abs(lhs - rhs) <= 1e-12 * max(abs(lhs), np.linalg.norm(cx) * np.linalg.norm(v))


@pytest.mark.gpu
def test_kernel_error_codes_leave_y_untouched(pm):
    import torch
    L = pm._lib
    x = torch.arange(24, dtype=torch.float64, device="cuda")
    y = torch.full((24,), 3.5, dtype=torch.float64, device="cuda")
    h = torch.ones(4, dtype=torch.float64, device="cuda")
    ARG, DT = 2002, 2001
    cases = [
        (dict(nh=0), ARG), (dict(nh=-1), ARG), (dict(off=-1), ARG), (dict(off=4), ARG),
        (dict(h=None), ARG), (dict(x=None), ARG), (dict(y=None), ARG), (dict(y="x"), ARG),
        (dict(dtype=L.C64), DT), (dict(dtype=L.BF16), DT), (dict(dtype=99), DT),
    ]
    assert_rejected(lambda a: c_conv(pm, a["x"], a["y"], (2, 3, 4), a["h"], a["nh"], a["off"], 0, a["dtype"]),
                    dict(x=x.data_ptr(), y=y.data_ptr(), h=h.data_ptr(), nh=4, off=1, dtype=L.F64), cases, y)
    for shape in ((0, 3, 4), (2, 0, 4), (2, 3, 0)):
        assert c_conv(pm, x.data_ptr(), y.data_ptr(), shape, h.data_ptr(), 4, 1, 0, L.F64) == 0
    torch.cuda.synchronize()
    assert torch.all(y == 3.5)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the operator
# ---------------------------------------------------------------------------------------------------------------
def blockdiag(pm, P, axis, h, off, dt):
    return pm.MPIBlockDiag([pm.local.Convolve1D((ny,) + mgc.DIMS[1:], h, offset=off, axis=axis, dtype=dt)
                            for ny in rows_of(P, mgc.DIMS[0])])


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_operator_vs_reference_fixtures(pm, case):
    """the inputs are exactly representable and every partial sum is exact in float32 too, so the operator must
    reproduce the reference's outputs bit for bit in every dtype"""
    P, axis, nh, off, dt = case
    h, x, y = mgc.case_inputs(nh, dt)
    Op = blockdiag(pm, P, axis, h, off, dt)
    got = host((Op @ pm.DistributedArray.to_dist(x)).asarray())
    gota = host((Op.H @ pm.DistributedArray.to_dist(y)).asarray())
    assert got.dtype == np.dtype(dt) and gota.dtype == np.dtype(dt)
    gy, gya = decode(GOLD, mgc.key(P, axis, nh, off), dt, mgc.ENC)
    np.testing.assert_array_equal(got, gy)
    np.testing.assert_array_equal(gota, gya)


@pytest.mark.gpu
def test_real_taps_on_complex_data_keep_the_imaginary_part(pm):
    import torch
    rng = np.random.default_rng(3)
    h = rng.standard_normal(9)
    for axis in (-1, 0):
        Cop = pm.local.Convolve1D((6, 40), h, offset=4, axis=axis)        # float64 operator
        x = rng.standard_normal(240) + 1j * rng.standard_normal(240)
        y = host(Cop.matvec(torch.as_tensor(x).cuda()))
        ya = host(Cop.rmatvec(torch.as_tensor(x).cuda()))
        assert y.dtype == np.complex128
        np.testing.assert_allclose(y, conv_ref(x.reshape(6, 40), h, 4, False, axis).ravel(), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(ya, conv_ref(x.reshape(6, 40), h, 4, True, axis).ravel(), rtol=1e-12, atol=1e-12)


@pytest.mark.gpu
def test_operator_argument_errors(pm):
    h = np.ones(5)
    for off in (-1, 5, 9):
        with pytest.raises(ValueError):
            pm.local.Convolve1D((4, 8), h, offset=off)
    with pytest.raises(ValueError):
        pm.local.Convolve1D((4, 8), h, method="overlap-add")
    with pytest.raises(NotImplementedError):
        pm.local.Convolve1D((4, 8), np.ones((4, 5)))
    with pytest.raises(NotImplementedError):
        pm.local.Convolve1D((4, 8), h + 1j)
    a = pm.local.Convolve1D((4, 8), h, offset=2, method="fft")
    b = pm.local.Convolve1D((4, 8), h, offset=2, method="direct")
    import torch
    x = torch.as_tensor(np.random.default_rng(0).standard_normal(32)).cuda()
    assert torch.equal(a.matvec(x), b.matvec(x))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["float64", "float32", "complex128"])
def test_operator_dottest(pm, dt):
    from pylops_mpi_b200.utils.dottest import dottest
    rng = np.random.default_rng(8)
    Op = blockdiag(pm, 2, -1, rng.standard_normal(13), 6, dt)
    n = Op.shape[0]
    u = rng.standard_normal(n) + (1j * rng.standard_normal(n) if dt == "complex128" else 0)
    v = rng.standard_normal(n) + (1j * rng.standard_normal(n) if dt == "complex128" else 0)
    u = pm.DistributedArray.to_dist(u.astype(dt))
    v = pm.DistributedArray.to_dist(v.astype(dt))
    assert dottest(Op, u, v, rtol=1e-5 if dt == "float32" else 1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
def test_reflectivity_ista_vs_reference(pm, P):
    wav, m, alpha = mgc.refl_inputs()
    assert alpha == float(GOLD["refl/alpha"])
    dims = [(ny,) + mgc.REFL_DIMS[1:] for ny in rows_of(P, mgc.REFL_DIMS[0])]
    DDiag = pm.MPIBlockDiag([pm.local.FirstDerivative(d, axis=-1) for d in dims])
    CDiag = pm.MPIBlockDiag([pm.local.Convolve1D(d, wav, offset=mgc.REFL_OFF, axis=-1) for d in dims])
    d = CDiag @ (DDiag @ pm.DistributedArray.to_dist(m))
    np.testing.assert_allclose(host(d.asarray()), GOLD["refl/d"], rtol=1e-12, atol=1e-12)
    x0 = pm.DistributedArray.to_dist(np.zeros_like(m))
    x, iiter, cost = pm.ista(CDiag, d, x0, niter=mgc.REFL_NITER, eps=mgc.REFL_EPS, alpha=alpha, tol=1e-10)
    assert iiter == int(GOLD[f"refl/P{P}/iiter"])
    np.testing.assert_allclose(cost, GOLD[f"refl/P{P}/cost"], rtol=1e-10)
    np.testing.assert_allclose(host(x.asarray()), GOLD[f"refl/P{P}/x"], rtol=1e-9, atol=1e-11)


@pytest.mark.gpu
@pytest.mark.parametrize("axis", [-1, 0])
def test_cgls_graph_replay_matches_step_loop(pm, axis):
    rng = np.random.default_rng(12)
    dims = (16, 24, 40)
    Op = pm.MPIBlockDiag([pm.local.Convolve1D(dims, rng.standard_normal(11), offset=5, axis=axis)])
    y = Op @ pm.DistributedArray.to_dist(rng.standard_normal(int(np.prod(dims))))
    assert_cgls_replay_matches_steps(pm, Op, y, pm.DistributedArray.to_dist(np.zeros(int(np.prod(dims)))), 25, 20)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["float32", "float64"])
@pytest.mark.parametrize("nh,off", [(1, 0), (41, 20), (8, 0), (8, 7)])
def test_axis_last_matches_torch_conv1d(pm, dt, nh, off):
    import torch
    rng = np.random.default_rng(nh)
    h = rng.standard_normal(nh)
    dims = (5, 8, 777)
    x = torch.as_tensor(rng.standard_normal(dims).astype(dt)).cuda()
    y = pm.local.Convolve1D(dims, h, offset=off, axis=-1, dtype=dt).matvec(x).reshape(dims)
    # y[i] = sum_k h[k] x[i + off - k] = cross-correlation of x with flip(h), padded nh-1-off in front, off behind
    w = torch.as_tensor(h[::-1].copy().astype(dt)).cuda().reshape(1, 1, nh)
    xp = torch.nn.functional.pad(x.reshape(-1, 1, dims[-1]), (nh - 1 - off, off))
    ref = torch.nn.functional.conv1d(xp, w).reshape(dims)
    tol = 1e-12 if dt == "float64" else 1e-4
    torch.testing.assert_close(y, ref, rtol=tol, atol=tol * np.abs(h).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [1, 2])
def test_multi_rank_fixtures(nproc):
    needs_gpus(nproc)
    run_on_ranks("test_convolve", nproc)


def on_ranks(pm, comm):
    """each rank's MPIBlockDiag([Convolve1D]) block against its slice of the gathered fixtures, and the reflectivity
    ISTA flow against its fixture"""
    rank, P = comm.Get_rank(), comm.Get_size()

    def block(dims_global):
        """this rank's rows of a global array split along axis 0: (local_shapes, flat slice, local dims)"""
        rows = rows_of(P, dims_global[0])
        plane = int(np.prod(dims_global[1:]))
        lo, hi = sum(rows[:rank]) * plane, sum(rows[:rank + 1]) * plane
        return [(r * plane,) for r in rows], slice(lo, hi), (rows[rank],) + tuple(dims_global[1:])

    def check(name, got, ref, rtol, atol):
        np.testing.assert_allclose(got, ref, rtol=rtol, atol=atol, err_msg=f"[rank {rank}] {name}")

    ls, sl, dims = block(mgc.DIMS)
    for (Pc, axis, nh, off, dt) in CASES:
        if Pc != P:
            continue
        h, x, v = mgc.case_inputs(nh, dt)
        Op = pm.MPIBlockDiag([pm.local.Convolve1D(dims, h, offset=off, axis=axis, dtype=dt)])
        gy, gya = decode(GOLD, mgc.key(P, axis, nh, off), dt, mgc.ENC)   # exact: the inputs are exactly representable
        name = f"{mgc.key(P, axis, nh, off)}/{dt}"
        np.testing.assert_array_equal(host((Op @ pm.DistributedArray.to_dist(x, local_shapes=ls)).local_array),
                                      gy[sl], err_msg=f"[rank {rank}] {name}/y")
        np.testing.assert_array_equal(host((Op.H @ pm.DistributedArray.to_dist(v, local_shapes=ls)).local_array),
                                      gya[sl], err_msg=f"[rank {rank}] {name}/ya")

    ls, sl, dims = block(mgc.REFL_DIMS)
    wav, m, alpha = mgc.refl_inputs()
    DDiag = pm.MPIBlockDiag([pm.local.FirstDerivative(dims, axis=-1)])
    CDiag = pm.MPIBlockDiag([pm.local.Convolve1D(dims, wav, offset=mgc.REFL_OFF, axis=-1)])
    d = CDiag @ (DDiag @ pm.DistributedArray.to_dist(m, local_shapes=ls))
    check("refl/d", host(d.local_array), GOLD["refl/d"][sl], 1e-12, 1e-12)
    x0 = pm.DistributedArray.to_dist(np.zeros_like(m), local_shapes=ls)
    x, iiter, cost = pm.ista(CDiag, d, x0, niter=mgc.REFL_NITER, eps=mgc.REFL_EPS, alpha=alpha, tol=1e-10)
    assert iiter == int(GOLD[f"refl/P{P}/iiter"])
    check("refl/cost", np.asarray(cost), GOLD[f"refl/P{P}/cost"], 1e-10, 0)
    check("refl/x", host(x.local_array), GOLD[f"refl/P{P}/x"][sl], 1e-9, 1e-11)
