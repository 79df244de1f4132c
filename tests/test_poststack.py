"""Rank-local PoststackLinearModelling and Transpose (pylops.avo.poststack / pylops.basicoperators inside
MPIBlockDiag, tutorials/poststack.py).

    PoststackLinearModelling(wav, nt0, spatdims) = Convolve1D(dims, wav, offset=len(wav)//2, axis=0)
                                                   * FirstDerivative(dims, axis=0, sampling=1, kind=kind)

CPU: refshim's restatements against that definition, and the fixtures of tests/golden/poststack_golden.npz (made by
make_golden_poststack.py: the reference's MPIBlockDiag and solvers over the restatements; operator inputs exactly
representable, so every dtype must match them bit for bit).  GPU: the fused b2_poststack_axis kernel through the C
ABI, against NumPy and bit for bit against the two-launch chain, and the operators through the public interface."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_poststack as mgp  # noqa: E402
from fixture_codec import decode, rows_of  # noqa: E402
from op_checks import (assert_cgls_replay_matches_steps, assert_rejected, device_input, guarded_twice, host,  # noqa: E402
                       needs_gpus, run_on_ranks)

GOLD = np.load(os.path.join(HERE, "golden", "poststack_golden.npz"), allow_pickle=False)
CASES = mgp.cases()
U32 = 2.0 ** -24
KINDS = {"centered": 2, "forward": 0}          # B2_FD_CENTERED, B2_FD_FORWARD


def conv_ref(x, h, off, adjoint=False):
    """Convolve1D along the last axis: y[i] = sum_k h[k] x[i + off - k] (adjoint: the transpose)"""
    h = np.asarray(h, dtype=np.float64)
    nh = h.size
    if adjoint:
        h, off = h[::-1], nh - 1 - off
    n = x.shape[-1]
    y = np.zeros(x.shape, dtype=np.result_type(x.dtype, np.float64))
    for k in range(nh):
        s = off - k
        lo, hi = max(0, -s), min(n, n - s)
        if hi > lo:
            y[..., lo:hi] += h[k] * x[..., lo + s:hi + s]
    return y


def deriv_ref(x, kind, adjoint=False):
    """FirstDerivative(edge=False, sampling=1) along the last axis (adjoint: the transpose)"""
    y = np.zeros(x.shape, dtype=np.result_type(x.dtype, np.float64))
    if kind == "centered":
        if not adjoint:
            y[..., 1:-1] = 0.5 * (x[..., 2:] - x[..., :-2])
        else:
            y[..., :-2] -= 0.5 * x[..., 1:-1]
            y[..., 2:] += 0.5 * x[..., 1:-1]
    else:
        if not adjoint:
            y[..., :-1] = x[..., 1:] - x[..., :-1]
        else:
            y[..., :-1] -= x[..., :-1]
            y[..., 1:] += x[..., :-1]
    return y


def post_ref(x, wav, kind, adjoint=False, axis=0, off=None):
    """C D x (adjoint D^T C^T x) along ``axis``"""
    off = len(wav) // 2 if off is None else off
    x = np.moveaxis(np.asarray(x), axis, -1)
    y = (conv_ref(deriv_ref(x, kind), wav, off) if not adjoint
         else deriv_ref(conv_ref(x, wav, off, True), kind, True))
    return np.moveaxis(y, -1, axis)


def refshim():
    path = os.path.join(HERE, "golden", "refshim")
    sys.path.insert(0, path)
    try:
        from pylops.avo.poststack import PoststackLinearModelling
        from pylops.basicoperators.transpose import Transpose
    finally:
        sys.path.remove(path)
    return PoststackLinearModelling, Transpose


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
def d_matrix(n, kind):
    D = np.zeros((n, n))
    for j in range(n):
        if kind == "centered" and 1 <= j <= n - 2:
            D[j, j - 1], D[j, j + 1] = -0.5, 0.5
        elif kind == "forward" and j <= n - 2:
            D[j, j], D[j, j + 1] = -1.0, 1.0
    return D


def c_matrix(n, h, off):
    C = np.zeros((n, n))
    for i in range(n):
        for j in range(n):
            if 0 <= i + off - j < len(h):
                C[i, j] = h[i + off - j]
    return C


@pytest.mark.parametrize("kind", ["centered", "forward"])
@pytest.mark.parametrize("nh", range(1, 8))
def test_refshim_poststack_is_c_times_d(kind, nh):
    PoststackLinearModelling, _ = refshim()
    wav = np.random.default_rng(nh).standard_normal(nh)
    for nt0, spatdims in ((1, None), (2, 3), (3, (2, 2)), (9, None), (30, 2)):
        Op = PoststackLinearModelling(wav, nt0=nt0, spatdims=spatdims, kind=kind)
        ns = int(np.prod(spatdims)) if spatdims is not None else 1
        assert Op.shape == (nt0 * ns, nt0 * ns) and Op.dtype == wav.dtype
        M1 = c_matrix(nt0, wav, nh // 2) @ d_matrix(nt0, kind)
        M = np.kron(M1, np.eye(ns))                         # time is axis 0: the slow index
        eye = np.eye(nt0 * ns)
        np.testing.assert_allclose(np.stack([Op.matvec(e) for e in eye], 1), M, rtol=0, atol=1e-13)
        np.testing.assert_allclose(np.stack([Op.H.matvec(e) for e in eye], 1), M.T, rtol=0, atol=1e-13)
        x = np.random.default_rng(0).standard_normal((nt0, ns))
        np.testing.assert_allclose(post_ref(x, wav, kind).ravel(), M @ x.ravel(), rtol=0, atol=1e-12)
        np.testing.assert_allclose(post_ref(x, wav, kind, True).ravel(), M.T @ x.ravel(), rtol=0, atol=1e-12)
    with pytest.raises(NotImplementedError):
        PoststackLinearModelling(wav, 5, kind="backward")


@pytest.mark.parametrize("dims,axes", [((3, 4, 5), (2, 0, 1)), ((3, 4, 5), (1, 2, 0)), ((6, 7), (1, 0)), ((5,), (0,))])
def test_transpose_and_its_adjoint(dims, axes):
    import torch
    from pylops_mpi_b200.local import Transpose
    _, RTranspose = refshim()
    x = np.random.default_rng(1).standard_normal(int(np.prod(dims)))
    ref = x.reshape(dims).transpose(axes).ravel()
    for Top in (Transpose(dims, axes), RTranspose(dims, axes)):
        y = Top.matvec(torch.as_tensor(x)) if isinstance(Top, Transpose) else Top.matvec(x)
        np.testing.assert_array_equal(np.asarray(y), ref)
        back = Top.rmatvec(y)
        np.testing.assert_array_equal(np.asarray(back), x)
        np.testing.assert_array_equal(np.asarray(Top.H.matvec(y)), x)
    T = Transpose(dims, axes)
    assert T.H.dims == T.dimsd and T.H.H.axes == T.axes and isinstance(T.H, Transpose)
    for bad in ((0, 0, 1), (0, 1), (0, 1, 3)):
        if len(dims) == 3:
            with pytest.raises(ValueError):
                Transpose(dims, bad)


def case_id(c):
    return f"{c[0]}/P{c[1]}/{c[2]}/nh{c[3]}/{c[4]}"


def test_poststack_fixture_inventory():
    assert len(CASES) == 2 * 3 * 2 * 4 * 2 + 2 * 3
    stored = set()
    for layout, P, kind, nh, dt in CASES:
        k = mgp.key(layout, P, kind, nh)
        for n in ("y", "ya", "yi", "yai")[:4 if dt == "complex128" else 2]:
            a = GOLD[f"{k}/{n}"]
            assert a.dtype == np.int16 and a.shape == (mgp.NY * mgp.NX * mgp.NT0,)
            stored.add(f"{k}/{n}")
    # native layout: one entry per P; tutorial layout does not depend on P; the complex cases add yi, yai
    assert len(stored) == (3 + 1) * (2 * 4 * 2 + 2)
    flows = {f"flow/P{P}/{f}/{k}" for P in (1, 2, 3) for f in ("iter", "ne", "reg") for k in ("x", "iiter", "cost")}
    for P in (1, 2, 3):
        for f in ("iter", "ne", "reg"):
            assert int(GOLD[f"flow/P{P}/{f}/iiter"]) == mgp.FLOW_NITER
            assert GOLD[f"flow/P{P}/{f}/x"].shape == (mgp.FLOW_NY * mgp.NX * mgp.NT0,)
    assert sorted(GOLD.files) == sorted(stored | flows | {"flow/d"})


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_fixtures_follow_the_definition(case):
    layout, P, kind, nh, dt = case
    wav, x, v = mgp.case_inputs(nh, dt)
    parts = np.cumsum([0] + [r * mgp.NX * mgp.NT0 for r in rows_of(P, mgp.NY)])
    fwd, adj = [], []
    for a, b, ny_r in zip(parts[:-1], parts[1:], rows_of(P, mgp.NY)):
        dims = mgp.block_dims(layout, ny_r)
        axis = 0 if layout == "native" else 2
        fwd.append(post_ref(x[a:b].reshape(dims), wav, kind, False, axis).ravel())
        adj.append(post_ref(v[a:b].reshape(dims), wav, kind, True, axis).ravel())
    gy, gya = decode(GOLD, mgp.key(layout, P, kind, nh), dt, mgp.ENC)
    np.testing.assert_array_equal(gy, np.concatenate(fwd))       # exact: every value is a multiple of 1/4
    np.testing.assert_array_equal(gya, np.concatenate(adj))


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernel through the C ABI
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


def c_post(pm, x, y, shape, h, nh, off, kind, adjoint, code):
    L = pm._lib
    return L.lib.b2_poststack_axis(L.ctx(), x, y, shape[0], shape[1], shape[2], h, nh, off, kind, adjoint, code,
                                   L.stream())


def run_kernel(pm, x_np, h_np, off, kind, adjoint, dt, misalign=False, guard=5):
    """apply through the C ABI into a guarded interior view; returns (y, guards intact, second apply bit-equal)"""
    x, h = device_input(x_np, dt, misalign), device_input(h_np, dt)
    code = pm._lib.F32 if dt == np.float32 else pm._lib.F64
    args = (x_np.shape, h.data_ptr(), h.numel(), off, KINDS[kind], int(adjoint), code)
    y, guards_ok, same = guarded_twice(lambda yp: c_post(pm, x.data_ptr(), yp, *args), x_np.size, dt, guard,
                                       int(misalign))
    return y.reshape(x_np.shape), guards_ok, same


def check_close(got, x, h, off, kind, adjoint, dt):
    ref = post_ref(x.astype(np.float64), h.astype(np.float64), kind, adjoint, 1, off)
    bnd = 2 * np.abs(h.astype(np.float64)).sum() * np.abs(x.astype(np.float64)).max()   # |D| <= 2, |C| <= |h|_1
    tol = (1e-12 * bnd) if dt == np.float64 else (4 * (h.size + 3) * U32 * bnd)
    err = np.abs(got.astype(np.float64) - ref)
    assert np.all(err <= tol), f"max err {err.max():.3e}, tol {tol:.3e}"


NHS = (1, 2, 5, 41, 300)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["centered", "forward"])
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("n_inner", [1, 3, 8], ids=["inner1", "inner3", "inner8"])
@pytest.mark.parametrize("nh", NHS)
def test_kernel_vs_numpy(pm, kind, dt, n_inner, nh):
    rng = np.random.default_rng(nh * 10 + n_inner)
    h = rng.standard_normal(nh).astype(dt)
    for n in sorted({1, 2, 3, max(1, nh - 1), 37, 4100}):
        n_outer = 3 if n * n_inner < 20000 else 1
        x = rng.standard_normal((n_outer, n, n_inner)).astype(dt)
        for off in sorted({0, nh // 2, nh - 1}):
            for adjoint in (False, True):
                for misalign in (False, True):
                    y, guards, same = run_kernel(pm, x, h, off, kind, adjoint, dt, misalign)
                    assert guards and same, (n, off, adjoint, misalign)
                    check_close(y, x, h, off, kind, adjoint, dt)


def chain(pm, x, shape, h, off, kind, adjoint, code):
    """the two-launch chain: b2_derivative_axis then b2_convolve_axis (adjoint: the reverse)"""
    import torch
    L = pm._lib
    t, y = torch.empty_like(x), torch.empty_like(x)
    d = lambda a, b: L.lib.b2_derivative_axis(L.ctx(), a.data_ptr(), b.data_ptr(), *shape, 1, KINDS[kind], 3, 0,  # noqa: E731
                                              1.0, int(adjoint), code, L.stream())
    c = lambda a, b: L.lib.b2_convolve_axis(L.ctx(), a.data_ptr(), b.data_ptr(), *shape, h.data_ptr(), h.numel(),  # noqa: E731
                                            off, int(adjoint), code, L.stream())
    assert (c(x, t) == 0 and d(t, y) == 0) if adjoint else (d(x, t) == 0 and c(t, y) == 0)
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["float32", "float64"])
@pytest.mark.parametrize("shape", [(3, 1000, 1), (2, 4100, 1), (4, 37, 1), (5, 1, 1), (5, 2, 1), (5, 3, 1),
                                   (3, 50, 3), (2, 70, 8), (2, 130, 64), (5, 2, 4), (1, 1024, 33)])
def test_kernel_equals_two_launch_chain_bitwise(pm, dt, shape):
    import torch
    code = pm._lib.F32 if dt == "float32" else pm._lib.F64
    rng = np.random.default_rng(shape[1])
    x = torch.as_tensor(rng.standard_normal(int(np.prod(shape))).astype(dt)).cuda()
    y = torch.empty_like(x)
    for nh in (1, 4, 41, 300):
        h = torch.as_tensor(rng.standard_normal(nh).astype(dt)).cuda()
        for kind in KINDS:
            for adjoint in (False, True):
                assert c_post(pm, x.data_ptr(), y.data_ptr(), shape, h.data_ptr(), nh, nh // 2, KINDS[kind],
                              int(adjoint), code) == 0
                ref = chain(pm, x, shape, h, nh // 2, kind, adjoint, code)
                torch.cuda.synchronize()
                assert torch.equal(y, ref), (nh, kind, adjoint, (y - ref).abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("n_inner", [1, 4])
def test_kernel_n_outer_beyond_grid_limit(pm, dt, n_inner):
    rng = np.random.default_rng(5)
    h = rng.standard_normal(7).astype(dt)
    x = rng.standard_normal((70001, 5, n_inner)).astype(dt)
    for kind in KINDS:
        for adjoint in (False, True):
            y, guards, same = run_kernel(pm, x, h, 3, kind, adjoint, dt)
            assert guards and same
            check_close(y, x, h, 3, kind, adjoint, dt)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["centered", "forward"])
@pytest.mark.parametrize("shape", [(4, 300, 1), (3, 2100, 1), (3, 50, 6), (2, 7, 16), (2, 200, 8)])
@pytest.mark.parametrize("nh", [5, 41, 130])
def test_kernel_adjoint_dot(pm, kind, shape, nh):
    rng = np.random.default_rng(11)
    h = rng.standard_normal(nh)
    x, v = rng.standard_normal(shape), rng.standard_normal(shape)
    cx, _, _ = run_kernel(pm, x, h, nh // 2, kind, False, np.float64)
    chv, _, _ = run_kernel(pm, v, h, nh // 2, kind, True, np.float64)
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
        (dict(kind=1), ARG), (dict(kind=3), ARG), (dict(kind=-1), ARG),
        (dict(dtype=L.C64), DT), (dict(dtype=L.BF16), DT), (dict(dtype=99), DT),
    ]
    assert_rejected(lambda a: c_post(pm, a["x"], a["y"], (2, 3, 4), a["h"], a["nh"], a["off"], a["kind"], 0, a["dtype"]),
                    dict(x=x.data_ptr(), y=y.data_ptr(), h=h.data_ptr(), nh=4, off=1, kind=2, dtype=L.F64), cases, y)
    for shape in ((0, 3, 4), (2, 0, 4), (2, 3, 0)):
        assert c_post(pm, x.data_ptr(), y.data_ptr(), shape, h.data_ptr(), 4, 1, 2, 0, L.F64) == 0
    torch.cuda.synchronize()
    assert torch.all(y == 3.5)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the operators
# ---------------------------------------------------------------------------------------------------------------
def local_op(pm, layout, ny_r, wav, kind):
    PPop = pm.local.PoststackLinearModelling(wav, nt0=mgp.NT0, spatdims=(ny_r, mgp.NX), kind=kind)
    if layout == "native":
        return PPop
    Top = pm.local.Transpose((ny_r, mgp.NX, mgp.NT0), (2, 0, 1))
    return Top.H @ PPop @ Top


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_operator_vs_reference_fixtures(pm, case):
    """exactly representable inputs: the operator must reproduce the reference's outputs bit for bit in every dtype"""
    layout, P, kind, nh, dt = case
    wav, x, v = mgp.case_inputs(nh, dt)
    ops = [local_op(pm, layout, r, wav, kind) for r in rows_of(P, mgp.NY)]
    assert all(type(op).__name__ == "PoststackLinearModelling" for op in ops)          # the fold
    Op = pm.MPIBlockDiag(ops, dtype=dt)
    got = host((Op @ pm.DistributedArray.to_dist(x)).asarray())
    gota = host((Op.H @ pm.DistributedArray.to_dist(v)).asarray())
    assert got.dtype == np.dtype(dt) and gota.dtype == np.dtype(dt)
    gy, gya = decode(GOLD, mgp.key(layout, P, kind, nh), dt, mgp.ENC)
    np.testing.assert_array_equal(got, gy)
    np.testing.assert_array_equal(gota, gya)


@pytest.mark.gpu
def test_real_wavelet_on_complex_data_keeps_the_imaginary_part(pm):
    import torch
    rng = np.random.default_rng(3)
    wav = rng.standard_normal(9)
    for spatdims in ((6, 5), None):
        Op = pm.local.PoststackLinearModelling(wav, nt0=40, spatdims=spatdims)
        n = Op.shape[0]
        x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        y = host(Op.matvec(torch.as_tensor(x).cuda()))
        ya = host(Op.rmatvec(torch.as_tensor(x).cuda()))
        assert y.dtype == np.complex128
        x3 = x.reshape((40,) + (spatdims or ()))
        np.testing.assert_allclose(y, post_ref(x3, wav, "centered").ravel(), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(ya, post_ref(x3, wav, "centered", True).ravel(), rtol=1e-12, atol=1e-12)


@pytest.mark.gpu
def test_operator_argument_errors(pm):
    wav = np.ones(5)
    for kw in (dict(explicit=True), dict(sparse=True), dict(kind="backward"), dict(kind="nope")):
        with pytest.raises(NotImplementedError):
            pm.local.PoststackLinearModelling(wav, 10, **kw)
    with pytest.raises(NotImplementedError):
        pm.local.PoststackLinearModelling(np.ones((4, 5)), 10)
    with pytest.raises(NotImplementedError):
        pm.local.PoststackLinearModelling(wav + 1j, 10)
    Op = pm.local.PoststackLinearModelling(wav.astype(np.float32), 10, 3)
    assert Op.dims == (10, 3) and Op.axis == 0 and Op.dtype == np.float32 and Op.shape == (30, 30)
    assert pm.local.PoststackLinearModelling(wav, 10, (3, 2)).dims == (10, 3, 2)
    with pytest.raises(ValueError):
        pm.local.Transpose((2, 3), (0, 0))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["float64", "float32", "complex128"])
def test_operator_dottest(pm, dt):
    from pylops_mpi_b200.utils.dottest import dottest
    rng = np.random.default_rng(8)
    wav = rng.standard_normal(13).astype("float32" if dt == "float32" else "float64")
    for layout in mgp.LAYOUTS:
        Op = pm.MPIBlockDiag([local_op(pm, layout, r, wav, "centered") for r in (3, 2)], dtype=dt)
        n = Op.shape[0]
        u = rng.standard_normal(n) + (1j * rng.standard_normal(n) if dt == "complex128" else 0)
        v = rng.standard_normal(n) + (1j * rng.standard_normal(n) if dt == "complex128" else 0)
        assert dottest(Op, pm.DistributedArray.to_dist(u.astype(dt)), pm.DistributedArray.to_dist(v.astype(dt)),
                       rtol=1e-5 if dt == "float32" else 1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["centered", "forward"])
def test_fold_is_one_operator_along_the_transposed_axis(pm, kind):
    import torch
    from pylops_mpi_b200.local import Transpose, PoststackLinearModelling, Convolve1D, FirstDerivative, \
        SecondDerivative, _LocalProduct
    rng = np.random.default_rng(4)
    wav = rng.standard_normal(41)
    ny, nx, nz = 3, 5, 64
    PPop = PoststackLinearModelling(wav, nt0=nz, spatdims=(ny, nx), kind=kind)
    Top = Transpose((ny, nx, nz), (2, 0, 1))
    a, b = (Top.H @ PPop) @ Top, Top.H @ (PPop @ Top)
    for f in (a, b, Top.H * PPop * Top):
        assert type(f) is PoststackLinearModelling and f.axis == 2 and f.dims == (ny, nx, nz)
    assert PPop.axis == 0 and PPop.dims == (nz, ny, nx)                   # the user's operator is unchanged
    x = torch.as_tensor(rng.standard_normal(ny * nx * nz)).cuda()
    unfolded = Top.rmatvec(PPop.matvec(Top.matvec(x)))
    unfolded_a = Top.rmatvec(PPop.rmatvec(Top.matvec(x)))
    torch.testing.assert_close(a.matvec(x), unfolded, rtol=1e-13, atol=1e-13)
    torch.testing.assert_close(a.rmatvec(x), unfolded_a, rtol=1e-13, atol=1e-13)
    ref = post_ref(host(x).reshape(ny, nx, nz), wav, kind, False, 2).ravel()
    np.testing.assert_allclose(host(a.matvec(x)), ref, rtol=1e-12, atol=1e-12)
    # other axis operators fold the same way; a product that is not T.H @ X @ T stays an (eager) product
    T2 = Transpose((4, 6, 8), (1, 2, 0))
    for X in (Convolve1D((6, 8, 4), wav[:5], offset=2, axis=1), FirstDerivative((6, 8, 4), axis=2),
              SecondDerivative((6, 8, 4), axis=0)):
        F = T2.H @ X @ T2
        assert type(F) is type(X) and F.axis == T2.axes[X.axis] and F.dims == (4, 6, 8)
        y = torch.as_tensor(rng.standard_normal(192)).cuda()
        torch.testing.assert_close(F.matvec(y), T2.rmatvec(X.matvec(T2.matvec(y))), rtol=1e-13, atol=1e-13)
    P = PPop @ Top
    assert isinstance(P, _LocalProduct) and P.shape == (ny * nx * nz,) * 2
    torch.testing.assert_close(P.matvec(x), PPop.matvec(Top.matvec(x)))
    torch.testing.assert_close(P.H.matvec(x), Top.rmatvec(PPop.rmatvec(x)))
    assert isinstance(Top @ PPop, _LocalProduct)                        # dims do not match the fold: no fold


def ricker(t, f0):
    """pylops.utils.wavelets.ricker, restated"""
    w = (1 - 2 * (np.pi * f0 * t) ** 2) * np.exp(-(np.pi * f0 * t) ** 2)
    return np.concatenate((np.flipud(w[1:]), w), axis=0)


def check_flow(name, P, x, iiter, cost):
    g = f"flow/P{P}/{name}"
    assert iiter == int(GOLD[f"{g}/iiter"])
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"{g}/cost"], rtol=1e-10)
    np.testing.assert_allclose(host(x.asarray()), GOLD[f"{g}/x"], rtol=1e-9, atol=1e-11)


@pytest.mark.gpu
def test_tutorial_poststack_line_for_line(pm):
    """tutorials/poststack.py at (6, 4, 33) on one rank, statement by statement (the model is a fixture input)"""
    import pylops_mpi_b200 as pylops_mpi
    from pylops_mpi_b200.local import PoststackLinearModelling, Transpose
    _, m3d_i, mback3d_i = mgp.flow_inputs()
    ny_i, nx, nz = m3d_i.shape
    ny = ny_i
    dt = 0.004
    t0 = np.arange(nz) * dt
    ntwav = 15
    wav = ricker(t0[:ntwav // 2 + 1], 15)
    assert np.array_equal(wav, mgp.flow_inputs()[0])

    m3d_dist = pylops_mpi.DistributedArray(global_shape=ny * nx * nz)
    m3d_dist[:] = m3d_i.flatten()
    mback3d_dist = pylops_mpi.DistributedArray(global_shape=ny * nx * nz)
    mback3d_dist[:] = mback3d_i.flatten()
    PPop = PoststackLinearModelling(wav, nt0=nz, spatdims=(ny_i, nx))
    Top = Transpose((ny_i, nx, nz), (2, 0, 1))
    BDiag = pylops_mpi.basicoperators.MPIBlockDiag(ops=[Top.H @ PPop @ Top, ])
    d_dist = BDiag @ m3d_dist
    np.testing.assert_allclose(host(d_dist.asarray()), GOLD["flow/d"], rtol=1e-12, atol=1e-12)

    minv3d_iter_dist, _, iiter, _, _, cost = pylops_mpi.optimization.basic.cgls(
        BDiag, d_dist, x0=mback3d_dist, niter=mgp.FLOW_NITER, show=False, tol=0.0)
    check_flow("iter", 1, minv3d_iter_dist, iiter, cost)

    epsR = 1e2
    LapOp = pylops_mpi.MPILaplacian(dims=(ny, nx, nz), axes=(0, 1, 2), weights=(1, 1, 1),
                                    sampling=(1, 1, 1), dtype=BDiag.dtype)
    NormEqOp = BDiag.H @ BDiag + epsR * LapOp.H @ LapOp
    dnorm_dist = BDiag.H @ d_dist
    minv3d_ne_dist, iiter, cost = pylops_mpi.optimization.basic.cg(NormEqOp, dnorm_dist, x0=mback3d_dist,
                                                                   niter=mgp.FLOW_NITER, show=False, tol=0.0)
    check_flow("ne", 1, minv3d_ne_dist, iiter, cost)

    StackOp = pylops_mpi.MPIStackedVStack([BDiag, np.sqrt(epsR) * LapOp])
    d0_dist = pylops_mpi.DistributedArray(global_shape=ny * nx * nz)
    d0_dist[:] = 0.
    dstack_dist = pylops_mpi.StackedDistributedArray([d_dist, d0_dist])
    minv3d_reg_dist, _, iiter, _, _, cost = pylops_mpi.optimization.basic.cgls(
        StackOp, dstack_dist, x0=mback3d_dist, niter=mgp.FLOW_NITER, show=False, tol=0.0)
    check_flow("reg", 1, minv3d_reg_dist, iiter, cost)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
def test_tutorial_flows_vs_reference(pm, P):
    """the three solves with the y rows of P ranks held as P blocks of one MPIBlockDiag"""
    wav, m3d, mback3d = mgp.flow_inputs()
    ny = rows_of(P, mgp.FLOW_NY)
    nx, nz = mgp.NX, mgp.NT0
    ops = []
    for ny_i in ny:
        PPop = pm.local.PoststackLinearModelling(wav, nt0=nz, spatdims=(ny_i, nx))
        Top = pm.local.Transpose((ny_i, nx, nz), (2, 0, 1))
        ops.append(Top.H @ PPop @ Top)
    BDiag = pm.MPIBlockDiag(ops)
    m = pm.DistributedArray.to_dist(m3d.ravel())
    x0 = pm.DistributedArray.to_dist(mback3d.ravel())
    d = BDiag @ m
    np.testing.assert_allclose(host(d.asarray()), GOLD["flow/d"], rtol=1e-12, atol=1e-12)
    x, _, iiter, _, _, cost = pm.cgls(BDiag, d, x0=x0, niter=mgp.FLOW_NITER, tol=0.0)
    check_flow("iter", P, x, iiter, cost)
    LapOp = pm.MPILaplacian(dims=(mgp.FLOW_NY, nx, nz), axes=(0, 1, 2), weights=(1, 1, 1), sampling=(1, 1, 1),
                            dtype=BDiag.dtype)
    x, iiter, cost = pm.cg(BDiag.H @ BDiag + mgp.FLOW_EPSR * LapOp.H @ LapOp, BDiag.H @ d, x0=x0,
                           niter=mgp.FLOW_NITER, tol=0.0)
    check_flow("ne", P, x, iiter, cost)
    zero = pm.DistributedArray.to_dist(np.zeros(m3d.size))
    x, _, iiter, _, _, cost = pm.cgls(pm.MPIStackedVStack([BDiag, np.sqrt(mgp.FLOW_EPSR) * LapOp]),
                                      pm.StackedDistributedArray([d, zero]), x0=x0, niter=mgp.FLOW_NITER, tol=0.0)
    check_flow("reg", P, x, iiter, cost)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", mgp.LAYOUTS)
def test_cgls_graph_replay_matches_step_loop(pm, layout):
    rng = np.random.default_rng(12)
    wav = rng.standard_normal(21)
    Op = pm.MPIBlockDiag([local_op(pm, layout, 24, wav, "centered")])
    n = Op.shape[0]
    y = Op @ pm.DistributedArray.to_dist(rng.standard_normal(n))
    assert_cgls_replay_matches_steps(pm, Op, y, pm.DistributedArray.to_dist(np.zeros(n)), 25, 20)


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [1, 2])
def test_multi_rank_fixtures(nproc):
    needs_gpus(nproc)
    run_on_ranks("test_poststack", nproc)


def on_ranks(pm, comm):
    """each rank's MPIBlockDiag block against its slice of the gathered fixtures, and the three solves of
    tutorials/poststack.py against their fixtures"""
    rank, P = comm.Get_rank(), comm.Get_size()

    def block(ny):
        """this rank's rows of y: (local_shapes, flat slice, local rows)"""
        rows = rows_of(P, ny)
        plane = mgp.NX * mgp.NT0
        lo, hi = sum(rows[:rank]) * plane, sum(rows[:rank + 1]) * plane
        return [(r * plane,) for r in rows], slice(lo, hi), rows[rank]

    def check(name, got, ref, rtol, atol):
        np.testing.assert_allclose(got, ref, rtol=rtol, atol=atol, err_msg=f"[rank {rank}] {name}")

    ls, sl, ny_r = block(mgp.NY)
    for (layout, Pc, kind, nh, dt) in CASES:
        if Pc != P:
            continue
        wav, x, v = mgp.case_inputs(nh, dt)
        Op = pm.MPIBlockDiag([local_op(pm, layout, ny_r, wav, kind)], dtype=dt)
        gy, gya = decode(GOLD, mgp.key(layout, P, kind, nh), dt, mgp.ENC)   # exact: exactly representable inputs
        name = f"{mgp.key(layout, P, kind, nh)}/{dt}"
        np.testing.assert_array_equal(host((Op @ pm.DistributedArray.to_dist(x, local_shapes=ls)).local_array),
                                      gy[sl], err_msg=f"[rank {rank}] {name}/y")
        np.testing.assert_array_equal(host((Op.H @ pm.DistributedArray.to_dist(v, local_shapes=ls)).local_array),
                                      gya[sl], err_msg=f"[rank {rank}] {name}/ya")

    ls, sl, ny_i = block(mgp.FLOW_NY)
    wav, m3d, mback3d = mgp.flow_inputs()
    nx, nz = mgp.NX, mgp.NT0
    PPop = pm.local.PoststackLinearModelling(wav, nt0=nz, spatdims=(ny_i, nx))
    Top = pm.local.Transpose((ny_i, nx, nz), (2, 0, 1))
    BDiag = pm.MPIBlockDiag([Top.H @ PPop @ Top])
    m = pm.DistributedArray.to_dist(m3d.ravel(), local_shapes=ls)
    x0 = pm.DistributedArray.to_dist(mback3d.ravel(), local_shapes=ls)
    d = BDiag @ m
    check("flow/d", host(d.local_array), GOLD["flow/d"][sl], 1e-12, 1e-12)

    def check_flow(name, x, iiter, cost):
        g = f"flow/P{P}/{name}"
        assert iiter == int(GOLD[f"{g}/iiter"])
        check(f"{g}/cost", np.asarray(cost), GOLD[f"{g}/cost"], 1e-10, 0)
        check(f"{g}/x", host(x.local_array), GOLD[f"{g}/x"][sl], 1e-9, 1e-11)

    x, _, iiter, _, _, cost = pm.cgls(BDiag, d, x0=x0, niter=mgp.FLOW_NITER, tol=0.0)
    check_flow("iter", x, iiter, cost)
    LapOp = pm.MPILaplacian(dims=(mgp.FLOW_NY, nx, nz), axes=(0, 1, 2), weights=(1, 1, 1), sampling=(1, 1, 1),
                            dtype=BDiag.dtype)
    x, iiter, cost = pm.cg(BDiag.H @ BDiag + mgp.FLOW_EPSR * LapOp.H @ LapOp, BDiag.H @ d, x0=x0,
                           niter=mgp.FLOW_NITER, tol=0.0)
    check_flow("ne", x, iiter, cost)
    zero = pm.DistributedArray.to_dist(np.zeros(m3d.size), local_shapes=ls)
    x, _, iiter, _, _, cost = pm.cgls(pm.MPIStackedVStack([BDiag, np.sqrt(mgp.FLOW_EPSR) * LapOp]),
                                      pm.StackedDistributedArray([d, zero]), x0=x0, niter=mgp.FLOW_NITER, tol=0.0)
    check_flow("reg", x, iiter, cost)
