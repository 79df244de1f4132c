"""Rank-local NonStationaryConvolve1D and the 2-D wavelet PoststackLinearModelling (pylops.signalprocessing /
pylops.avo.poststack inside MPIBlockDiag).

    h_j = hs[l] interpolated linearly between the filters at ih (first / last filter outside them)
    forward y[i] = sum_j h_j[hc + i - j] x[j],  adjoint the transpose
    PoststackLinearModelling(wav (nt0, nwav)) = C D,  C[i, j] = wav[j, nwav // 2 + i - j]

CPU: refshim's restatements against that definition and against each other, and the fixtures of
tests/golden/nsconvolve_golden.npz (made by make_golden_nsconvolve.py: the reference's MPIBlockDiag and solvers over the
restatements; operator inputs exactly representable, so every dtype must match them bit for bit).  GPU: the
b2_nsconvolve_axis / b2_nspoststack_axis kernels through the C ABI, and the operators through the public interface."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_nsconvolve as mgn  # noqa: E402
import make_golden_poststack as mgp  # noqa: E402
from fixture_codec import decode, rows_of  # noqa: E402
from op_checks import assert_cgls_replay_matches_steps, assert_rejected, device_input, guarded_twice, host  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "nsconvolve_golden.npz"), allow_pickle=False)
U32 = 2.0 ** -24
KINDS = {"centered": 2, "forward": 0}          # B2_FD_CENTERED, B2_FD_FORWARD


def refshim():
    path = os.path.join(HERE, "golden", "refshim")
    sys.path.insert(0, path)
    try:
        from pylops.signalprocessing.nonstatconvolve1d import NonStationaryConvolve1D
        from pylops.utils.signalprocessing import nonstationary_convmtx
        from pylops.avo.poststack_nonstationary import PoststackLinearModelling
    finally:
        sys.path.remove(path)
    return NonStationaryConvolve1D, nonstationary_convmtx, PoststackLinearModelling


def interp(hs, j, oh, dh):
    """h_j by the definition: pylops' _interpolate_h in the dtype of hs"""
    NS, _, _ = refshim()
    return np.asarray(NS._interpolate_h(hs, j, oh, dh, hs.shape[0]))


_NS_MATRICES = {}


def ns_matrix(hs, oh, dh, hc, n):
    """M[i, j] = h_j[hc + i - j] in float64 (h_j interpolated in the dtype of hs)"""
    key = (hs.tobytes(), hs.dtype.str, hs.shape, oh, dh, hc, n)
    if key not in _NS_MATRICES:
        _NS_MATRICES[key] = _ns_matrix(hs, oh, dh, hc, n)
    return _NS_MATRICES[key]


def _ns_matrix(hs, oh, dh, hc, n):
    M = np.zeros((n, n))
    nh = hs.shape[1]
    for j in range(n):
        h = interp(hs, j, oh, dh).astype(np.float64)
        for i in range(n):
            if 0 <= hc + i - j < nh:
                M[i, j] = h[hc + i - j]
    return M


def d_matrix(n, kind):
    D = np.zeros((n, n))
    for j in range(n):
        if kind == "centered" and 1 <= j <= n - 2:
            D[j, j - 1], D[j, j + 1] = -0.5, 0.5
        elif kind == "forward" and j <= n - 2:
            D[j, j], D[j, j + 1] = -1.0, 1.0
    return D


def along(M, x, axis):
    """apply the (n, n) matrix M along ``axis`` of x"""
    x = np.moveaxis(np.asarray(x), axis, 0)
    y = np.tensordot(M, x, axes=(1, 0))
    return np.moveaxis(y, 0, axis)


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nh", [1, 3, 5, 9])
@pytest.mark.parametrize("nf,dh,oh", [(1, 1, 0), (1, 1, 4), (2, 3, 1), (3, 2, 2), (4, 5, 0)])
def test_refshim_restatement_is_the_definition(nh, nf, dh, oh):
    NS, _, _ = refshim()
    rng = np.random.default_rng(nh * 100 + nf)
    hs = rng.standard_normal((nf, nh))
    ih = oh + dh * np.arange(nf)
    for dims, axis in (((23,), 0), ((4, 23), -1), ((23, 3), 0), ((2, 23, 2), 1)):
        Op = NS(dims, hs, ih, axis=axis)
        n = dims[axis]
        M = ns_matrix(hs, oh, dh, nh // 2, n)
        x = rng.standard_normal(dims)
        np.testing.assert_allclose(Op.matvec(x.ravel()), along(M, x, axis).ravel(), rtol=0, atol=1e-12)
        np.testing.assert_allclose(Op.rmatvec(x.ravel()), along(M.T, x, axis).ravel(), rtol=0, atol=1e-12)
    # the interpolation: exact weights between the filters, the end filters outside them
    for j in range(40):
        v = (j - oh) / dh
        lo = min(max(int(np.floor(v)), 0), nf - 1)
        if v <= 0 or lo == nf - 1:
            np.testing.assert_array_equal(interp(hs, j, oh, dh), hs[0] if v <= 0 else hs[nf - 1])
        else:
            w = v - lo
            np.testing.assert_array_equal(interp(hs, j, oh, dh), (1 - w) * hs[lo] + w * hs[lo + 1])
    for bad in (dict(hs=np.ones((nf, 4))), dict(ih=ih[:-1] if nf > 1 else [0, 1]), dict(ih=ih - oh - 1),
                dict(ih=ih + 23)):
        kw = dict(hs=hs if nh % 2 else np.ones((nf, 3)), ih=ih)
        kw.update(bad)
        with pytest.raises(ValueError):
            NS((23,), kw["hs"], kw["ih"])


@pytest.mark.parametrize("nh", [1, 3, 7])
def test_nonstationary_convolve_equals_the_poststack_convolution(nh):
    """pylops' two definitions agree: NonStationaryConvolve1D with one filter per sample is nonstationary_convmtx"""
    NS, convmtx, Post = refshim()
    for n in (1, 2, 9, 30):
        wav = np.random.default_rng(n + nh).standard_normal((n, nh))
        C = convmtx(wav, n, hc=nh // 2, pad=(n, n))
        Op = NS((n,), wav, np.arange(n))
        np.testing.assert_array_equal(np.stack([Op.matvec(e) for e in np.eye(n)], 1), C)
        np.testing.assert_array_equal(C, ns_matrix(wav, 0, 1, nh // 2, n))
        for kind in KINDS:
            P = Post(wav, nt0=n, spatdims=(2, 3), kind=kind)
            M = np.kron(C @ d_matrix(n, kind), np.eye(6))
            np.testing.assert_allclose(np.stack([P.matvec(e) for e in np.eye(6 * n)], 1), M, rtol=0, atol=1e-13)
            np.testing.assert_allclose(np.stack([P.rmatvec(e) for e in np.eye(6 * n)], 1), M.T, rtol=0, atol=1e-13)
    with pytest.raises(ValueError):
        Post(np.ones((4, 3)), nt0=5)


def test_nsconvolve_fixture_inventory():
    stored = set()
    for P, axis, nh, nf, dh, dt in mgn.ns_cases():
        k = mgn.ns_key(P, axis, nh, nf, dh)
        for n in ("y", "ya", "yi", "yai")[:4 if dt == "complex128" else 2]:
            assert GOLD[f"{k}/{n}"].dtype == np.int16 and GOLD[f"{k}/{n}"].shape == (int(np.prod(mgn.DIMS)),)
            stored.add(f"{k}/{n}")
    assert len(stored) == (3 + 1) * (2 * len(mgn.ns_configs()) + 2)
    post = set()
    for layout, P, kind, nw, dt in mgn.post_cases():
        k = mgn.post_key(layout, P, kind, nw)
        for n in ("y", "ya", "yi", "yai")[:4 if dt == "complex128" else 2]:
            assert GOLD[f"{k}/{n}"].dtype == np.int16 and GOLD[f"{k}/{n}"].shape == (mgn.NY * mgn.NX * mgn.NT0,)
            post.add(f"{k}/{n}")
    assert len(post) == (3 + 1) * (2 * 4 * 2 + 2)
    flows = {f"{f}/P{P}/{k}" for f in ("flow", "ista") for P in (1, 2, 3) for k in ("x", "iiter", "cost")}
    assert sorted(GOLD.files) == sorted(stored | post | flows | {"flow/d", "ista/d", "ista/alpha"})
    for P in (1, 2, 3):
        assert int(GOLD[f"flow/P{P}/iiter"]) == mgn.FLOW_NITER and int(GOLD[f"ista/P{P}/iiter"]) <= mgn.ISTA_NITER


def ns_case_id(c):
    return f"P{c[0]}/ax{c[1]}/nh{c[2]}/nf{c[3]}/dh{c[4]}/{c[5]}"


def post_case_id(c):
    return f"{c[0]}/P{c[1]}/{c[2]}/nw{c[3]}/{c[4]}"


def ns_blocks(P):
    return [(r,) + mgn.DIMS[1:] for r in rows_of(P, mgn.DIMS[0])]


@pytest.mark.parametrize("case", mgn.ns_cases(), ids=[ns_case_id(c) for c in mgn.ns_cases()])
def test_ns_fixtures_follow_the_restatement(case):
    NS, _, _ = refshim()
    P, axis, nh, nf, dh, dt = case
    hs, ih, x, v = mgn.ns_inputs(nh, nf, dh, dt)
    fwd, adj, a = [], [], 0
    for dims in ns_blocks(P):
        b = a + int(np.prod(dims))
        Op = NS(dims, hs, ih, axis=axis, dtype=dt)
        fwd.append(Op.matvec(x[a:b]))
        adj.append(Op.rmatvec(v[a:b]))
        a = b
    gy, gya = decode(GOLD, mgn.ns_key(P, axis, nh, nf, dh), dt, mgn.ENC)
    np.testing.assert_array_equal(np.concatenate(fwd), gy)
    np.testing.assert_array_equal(np.concatenate(adj), gya)


@pytest.mark.parametrize("case", mgn.post_cases(), ids=[post_case_id(c) for c in mgn.post_cases()])
def test_post_fixtures_follow_the_definition(case):
    layout, P, kind, nw, dt = case
    wav, x, v = mgn.post_inputs(nw, dt)
    M = ns_matrix(wav.astype(np.float64), 0, 1, nw // 2, mgn.NT0) @ d_matrix(mgn.NT0, kind)
    axis = 0 if layout == "native" else 2
    fwd, adj, a = [], [], 0
    for r in rows_of(P, mgp.NY):
        dims = mgp.block_dims(layout, r)
        b = a + int(np.prod(dims))
        fwd.append(along(M, x[a:b].reshape(dims), axis).ravel())
        adj.append(along(M.T, v[a:b].reshape(dims), axis).ravel())
        a = b
    gy, gya = decode(GOLD, mgn.post_key(layout, P, kind, nw), dt, mgn.ENC)
    np.testing.assert_array_equal(np.concatenate(fwd), gy)
    np.testing.assert_array_equal(np.concatenate(adj), gya)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernels through the C ABI
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


def c_ns(pm, x, y, shape, hs, nf, nh, hc, oh, dh, adjoint, code, kind=None):
    L = pm._lib
    if kind is None:
        return L.lib.b2_nsconvolve_axis(L.ctx(), x, y, *shape, hs, nf, nh, hc, oh, dh, adjoint, code, L.stream())
    return L.lib.b2_nspoststack_axis(L.ctx(), x, y, *shape, hs, nf, nh, hc, oh, dh, kind, adjoint, code, L.stream())


def run_kernel(pm, x_np, hs_np, hc, oh, dh, adjoint, dt, kind=None, misalign=False, guard=5):
    """apply through the C ABI into a guarded interior view; returns (y, guards intact, second apply bit-equal)"""
    x, hs = device_input(x_np, dt, misalign), device_input(hs_np, dt)
    code = pm._lib.F32 if dt == np.float32 else pm._lib.F64
    args = (x_np.shape, hs.data_ptr(), hs_np.shape[0], hs_np.shape[1], hc, oh, dh, int(adjoint), code,
            None if kind is None else KINDS[kind])
    y, guards_ok, same = guarded_twice(lambda yp: c_ns(pm, x.data_ptr(), yp, *args), x_np.size, dt, guard,
                                       int(misalign))
    return y.reshape(x_np.shape), guards_ok, same


def check_close(got, x, hs, hc, oh, dh, adjoint, dt, kind=None):
    """componentwise: |got - ref| <= c (nh + 3) u (|C| |D| |x|) against the float64 product of the definition"""
    n = x.shape[1]
    C = ns_matrix(hs.astype(dt), oh, dh, hc, n)
    D = d_matrix(n, kind) if kind is not None else np.eye(n)
    M, B = C @ D, np.abs(C) @ np.abs(D)
    ref = along(M.T if adjoint else M, x.astype(np.float64), 1)
    bnd = along(B.T if adjoint else B, np.abs(x.astype(np.float64)), 1)
    tol = (1e-12 * bnd) if dt == np.float64 else (4 * (hs.shape[1] + 3) * U32 * bnd)
    err = np.abs(got.astype(np.float64) - ref)
    assert np.all(err <= tol), f"max err {err.max():.3e}, excess {(err - tol).max():.3e}"


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("n_inner", [1, 3, 40], ids=["inner1", "inner3", "inner40"])
@pytest.mark.parametrize("nh", [1, 5, 41, 101])
def test_kernel_vs_numpy(pm, dt, n_inner, nh):
    rng = np.random.default_rng(nh * 10 + n_inner)
    for n in sorted({1, 2, 7, max(1, nh - 1), 130}):
        for nf, dh, oh in ((1, 1, 0), (3, 2, 1), (4, 37, 5)):
            hs = rng.standard_normal((nf, nh)).astype(dt)
            x = rng.standard_normal((2, n, n_inner)).astype(dt)
            for hc in sorted({0, nh // 2, nh - 1}):
                for adjoint in (False, True):
                    for kind in (None, "centered", "forward"):
                        misalign = adjoint
                        y, guards, same = run_kernel(pm, x, hs, hc, oh, dh, adjoint, dt, kind, misalign)
                        assert guards and same, (n, nf, hc, adjoint, kind)
                        check_close(y, x, hs, hc, oh, dh, adjoint, dt, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("shape", [(70001, 5, 4), (3, 1, 1), (3, 1, 5), (100000, 3, 1)])
def test_kernel_large_and_degenerate_shapes(pm, dt, shape):
    rng = np.random.default_rng(5)
    hs = rng.standard_normal((2, 7)).astype(dt)
    x = rng.standard_normal(shape).astype(dt)
    for kind in (None, "centered"):
        for adjoint in (False, True):
            y, guards, same = run_kernel(pm, x, hs, 3, 0, 2, adjoint, dt, kind)
            assert guards and same
            check_close(y, x, hs, 3, 0, 2, adjoint, dt, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("dh", [3, 5, 7])
@pytest.mark.parametrize("n_inner", [1, 2])
def test_interpolated_filters_are_pylops_bits(pm, dt, dh, n_inner):
    """unit vectors e_j, one line each: column j of the operator is h_j exactly"""
    rng = np.random.default_rng(dh)
    n, nh, nf, oh = 50, 9, 5, 4
    hs = rng.standard_normal((nf, nh)).astype(dt)
    eye = np.repeat(np.eye(n, dtype=dt)[:, :, None], n_inner, axis=2)       # line j holds e_j
    y, _, _ = run_kernel(pm, eye, hs, nh // 2, oh, dh, False, dt)
    for j in range(n):
        h = interp(hs, j, oh, dh)
        assert h.dtype == np.dtype(dt)
        col = np.zeros(n, dtype=dt)
        lo, hi = max(0, j - nh // 2), min(n, j + nh // 2 + 1)
        col[lo:hi] = h[lo - j + nh // 2:hi - j + nh // 2]
        for c in range(n_inner):
            np.testing.assert_array_equal(y[j, :, c], col, err_msg=f"j={j}")


def chain(pm, x, shape, hs, nf, nh, hc, oh, dh, kind, adjoint, code):
    """the two-launch chain: b2_derivative_axis then b2_nsconvolve_axis (adjoint: the reverse)"""
    import torch
    L = pm._lib
    t, y = torch.empty_like(x), torch.empty_like(x)
    d = lambda a, b: L.lib.b2_derivative_axis(L.ctx(), a.data_ptr(), b.data_ptr(), *shape, 1, KINDS[kind], 3, 0,  # noqa: E731
                                              1.0, int(adjoint), code, L.stream())
    c = lambda a, b: c_ns(pm, a.data_ptr(), b.data_ptr(), shape, hs.data_ptr(), nf, nh, hc, oh, dh,  # noqa: E731
                          int(adjoint), code)
    assert (c(x, t) == 0 and d(t, y) == 0) if adjoint else (d(x, t) == 0 and c(t, y) == 0)
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["float32", "float64"])
@pytest.mark.parametrize("shape", [(3, 1000, 1), (2, 130, 1), (5, 1, 1), (5, 2, 1), (3, 50, 3), (2, 70, 8),
                                   (2, 130, 64), (5, 2, 4), (1, 200, 33)])
def test_fused_poststack_equals_two_launch_chain_bitwise(pm, dt, shape):
    import torch
    code = pm._lib.F32 if dt == "float32" else pm._lib.F64
    rng = np.random.default_rng(shape[1])
    x = torch.as_tensor(rng.standard_normal(int(np.prod(shape))).astype(dt)).cuda()
    y = torch.empty_like(x)
    n = shape[1]
    for nh in (1, 4, 41, 60):
        hs = torch.as_tensor(rng.standard_normal((n, nh)).astype(dt)).cuda()
        for kind in KINDS:
            for adjoint in (False, True):
                assert c_ns(pm, x.data_ptr(), y.data_ptr(), shape, hs.data_ptr(), n, nh, nh // 2, 0, 1, int(adjoint),
                            code, KINDS[kind]) == 0
                ref = chain(pm, x, shape, hs, n, nh, nh // 2, 0, 1, kind, adjoint, code)
                torch.cuda.synchronize()
                assert torch.equal(y, ref), (nh, kind, adjoint, (y - ref).abs().max().item())


@pytest.mark.gpu
def test_kernel_error_codes_leave_y_untouched(pm):
    import torch
    L = pm._lib
    x = torch.arange(24, dtype=torch.float64, device="cuda")
    y = torch.full((24,), 3.5, dtype=torch.float64, device="cuda")
    hs = torch.ones(8, dtype=torch.float64, device="cuda")
    ARG, DT = 2002, 2001
    cases = [
        (dict(nf=0), ARG), (dict(nh=0), ARG), (dict(nh=-1), ARG), (dict(hc=-1), ARG), (dict(hc=4), ARG),
        (dict(dh=0), ARG), (dict(dh=-2), ARG), (dict(hs=None), ARG), (dict(x=None), ARG), (dict(y=None), ARG),
        (dict(y="x"), ARG), (dict(shape=(0, 3, 4)), ARG), (dict(shape=(2, 0, 4)), ARG), (dict(shape=(2, 3, 0)), ARG),
        (dict(dtype=L.C64), DT), (dict(dtype=L.BF16), DT), (dict(dtype=99), DT),
    ]
    for post in (False, True):
        assert_rejected(
            lambda a: c_ns(pm, a["x"], a["y"], a["shape"], a["hs"], a["nf"], a["nh"], a["hc"], 0, a["dh"], 0, a["dtype"],
                           a["kind"] if post else None),
            dict(x=x.data_ptr(), y=y.data_ptr(), hs=hs.data_ptr(), nf=2, nh=4, hc=1, dh=1, kind=2, dtype=L.F64,
                 shape=(2, 3, 4)),
            cases + ([(dict(kind=1), ARG), (dict(kind=3), ARG), (dict(kind=-1), ARG)] if post else []), y)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the operators
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", mgn.ns_cases(), ids=[ns_case_id(c) for c in mgn.ns_cases()])
def test_ns_operator_vs_reference_fixtures(pm, case):
    P, axis, nh, nf, dh, dt = case
    hs, ih, x, v = mgn.ns_inputs(nh, nf, dh, dt)
    Op = pm.MPIBlockDiag([pm.local.NonStationaryConvolve1D(d, hs, ih, axis=axis, dtype=hs.dtype) for d in ns_blocks(P)],
                         dtype=dt)
    got = host((Op @ pm.DistributedArray.to_dist(x)).asarray())
    gota = host((Op.H @ pm.DistributedArray.to_dist(v)).asarray())
    assert got.dtype == np.dtype(dt) and gota.dtype == np.dtype(dt)
    gy, gya = decode(GOLD, mgn.ns_key(P, axis, nh, nf, dh), dt, mgn.ENC)
    np.testing.assert_array_equal(got, gy)
    np.testing.assert_array_equal(gota, gya)


def local_post(pm, layout, ny_r, wav, kind):
    PPop = pm.local.PoststackLinearModelling(wav, nt0=mgn.NT0, spatdims=(ny_r, mgn.NX), kind=kind)
    if layout == "native":
        return PPop
    Top = pm.local.Transpose((ny_r, mgn.NX, mgn.NT0), (2, 0, 1))
    return Top.H @ PPop @ Top


@pytest.mark.gpu
@pytest.mark.parametrize("case", mgn.post_cases(), ids=[post_case_id(c) for c in mgn.post_cases()])
def test_post_operator_vs_reference_fixtures(pm, case):
    layout, P, kind, nw, dt = case
    wav, x, v = mgn.post_inputs(nw, dt)
    ops = [local_post(pm, layout, r, wav, kind) for r in rows_of(P, mgp.NY)]
    assert all(type(op).__name__ == "PoststackLinearModelling" and op.nonstationary for op in ops)   # the fold
    Op = pm.MPIBlockDiag(ops, dtype=dt)
    got = host((Op @ pm.DistributedArray.to_dist(x)).asarray())
    gota = host((Op.H @ pm.DistributedArray.to_dist(v)).asarray())
    gy, gya = decode(GOLD, mgn.post_key(layout, P, kind, nw), dt, mgn.ENC)
    np.testing.assert_array_equal(got, gy)
    np.testing.assert_array_equal(gota, gya)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["float64", "float32", "complex128"])
def test_operator_dottest(pm, dt):
    from pylops_mpi_b200.utils.dottest import dottest
    rng = np.random.default_rng(8)
    rdt = "float32" if dt == "float32" else "float64"
    hs = rng.standard_normal((3, 13)).astype(rdt)
    wav = rng.standard_normal((mgn.NT0, 12)).astype(rdt)
    ops = [pm.MPIBlockDiag([pm.local.NonStationaryConvolve1D((r, 30), hs, [2, 12, 22], axis=ax, dtype=rdt)
                            for r in (31, 30)], dtype=dt) for ax in (0, 1)]
    ops += [pm.MPIBlockDiag([local_post(pm, layout, r, wav, "centered") for r in (3, 2)], dtype=dt)
            for layout in mgp.LAYOUTS]
    for Op in ops:
        n = Op.shape[0]
        u = rng.standard_normal(n) + (1j * rng.standard_normal(n) if dt == "complex128" else 0)
        v = rng.standard_normal(n) + (1j * rng.standard_normal(n) if dt == "complex128" else 0)
        assert dottest(Op, pm.DistributedArray.to_dist(u.astype(dt)), pm.DistributedArray.to_dist(v.astype(dt)),
                       rtol=1e-5 if dt == "float32" else 1e-12)


@pytest.mark.gpu
def test_real_taps_on_complex_data_keep_the_imaginary_part(pm):
    import torch
    rng = np.random.default_rng(3)
    hs = rng.standard_normal((3, 9))
    wav = rng.standard_normal((40, 6))
    for Op, M, axis, shape in (
            (pm.local.NonStationaryConvolve1D((40, 6), hs, [3, 13, 23], axis=0), ns_matrix(hs, 3, 10, 4, 40), 0, (40, 6)),
            (pm.local.NonStationaryConvolve1D((6, 40), hs, [3, 13, 23]), ns_matrix(hs, 3, 10, 4, 40), 1, (6, 40)),
            (pm.local.PoststackLinearModelling(wav, nt0=40, spatdims=5), ns_matrix(wav, 0, 1, 3, 40) @
             d_matrix(40, "centered"), 0, (40, 5))):
        n = Op.shape[0]
        x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        y = host(Op.matvec(torch.as_tensor(x).cuda()))
        ya = host(Op.rmatvec(torch.as_tensor(x).cuda()))
        assert y.dtype == np.complex128
        np.testing.assert_allclose(y, along(M, x.reshape(shape), axis).ravel(), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(ya, along(M.T, x.reshape(shape), axis).ravel(), rtol=1e-12, atol=1e-12)


@pytest.mark.gpu
def test_operator_argument_errors(pm):
    NSC = pm.local.NonStationaryConvolve1D
    hs = np.ones((3, 5))
    for args in (((20,), np.ones((3, 4)), [2, 6, 10]),          # even nh
                 ((20,), hs, [2, 6, 11]),                       # irregular
                 ((20,), hs, [2, 6]),                           # len(ih) != nfilt
                 ((20,), hs, [-1, 3, 7]), ((20,), hs, [10, 15, 20]),   # outside [0, n)
                 ((20,), hs, [10, 6, 2]),                       # decreasing
                 ((20,), np.ones(5), [2])):                     # not a bank
        with pytest.raises(ValueError):
            NSC(*args)
    with pytest.raises(NotImplementedError):
        NSC((20,), hs + 1j, [2, 6, 10])
    with pytest.raises(NotImplementedError):
        pm.local.PoststackLinearModelling(np.ones((10, 5)) + 1j, 10)
    with pytest.raises(NotImplementedError):                    # first dimension is not nt0
        pm.local.PoststackLinearModelling(np.ones((4, 5)), 10)
    with pytest.raises(NotImplementedError):
        pm.local.Convolve1D(10, np.ones((2, 3)))
    Op = NSC((4, 20), hs.astype(np.float32), [2, 6, 10], axis=1, dtype="float32")
    assert Op.dims == (4, 20) and Op.axis == 1 and Op.dtype == np.float32 and Op.shape == (80, 80)
    assert (Op.oh, Op.dh, Op.hc, Op.nfilt, Op.nh) == (2, 4, 2, 3, 5)
    assert NSC((20,), hs[:1], [7]).dh == 1
    P = pm.local.PoststackLinearModelling(np.ones((10, 4), dtype=np.float32), 10, (3, 2))
    assert P.nonstationary and P.dims == (10, 3, 2) and P.dtype == np.float32 and P.offset == 2


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["ns_axis0", "ns_axis1", "post_native", "post_tut"])
def test_cgls_graph_replay_matches_step_loop(pm, which):
    rng = np.random.default_rng(12)
    if which.startswith("ns"):
        op = pm.local.NonStationaryConvolve1D((64, 48), rng.standard_normal((4, 21)), [3, 13, 23, 33],
                                              axis=int(which[-1]))
    else:
        op = local_post(pm, which[5:], 24, rng.standard_normal((mgn.NT0, 21)), "centered")
    Op = pm.MPIBlockDiag([op])
    n = Op.shape[0]
    y = Op @ pm.DistributedArray.to_dist(rng.standard_normal(n))
    assert_cgls_replay_matches_steps(pm, Op, y, pm.DistributedArray.to_dist(np.zeros(n)), 25, 20)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
def test_poststack_flow_with_time_varying_wavelet_vs_reference(pm, P):
    """tutorials/poststack.py's modelling and cgls, one Ricker wavelet per time sample, y rows of P ranks as P blocks"""
    wav, m3d, mback3d = mgn.flow_inputs()
    nx, nz = mgn.NX, mgn.NT0
    ops = []
    for ny_i in rows_of(P, mgn.FLOW_NY):
        PPop = pm.local.PoststackLinearModelling(wav, nt0=nz, spatdims=(ny_i, nx))
        Top = pm.local.Transpose((ny_i, nx, nz), (2, 0, 1))
        ops.append(Top.H @ PPop @ Top)
    BDiag = pm.MPIBlockDiag(ops)
    d = BDiag @ pm.DistributedArray.to_dist(m3d.ravel())
    np.testing.assert_allclose(host(d.asarray()), GOLD["flow/d"], rtol=1e-12, atol=1e-12)
    x, _, iiter, _, _, cost = pm.cgls(BDiag, d, x0=pm.DistributedArray.to_dist(mback3d.ravel()),
                                      niter=mgn.FLOW_NITER, tol=0.0)
    assert iiter == int(GOLD[f"flow/P{P}/iiter"])
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"flow/P{P}/cost"], rtol=1e-10)
    np.testing.assert_allclose(host(x.asarray()), GOLD[f"flow/P{P}/x"], rtol=1e-9, atol=1e-11)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
def test_ista_on_nonstationary_convolution_vs_reference(pm, P):
    hs, ih, m, alpha = mgn.ista_inputs()
    assert alpha == float(GOLD["ista/alpha"])
    dims = [(ny,) + mgn.ISTA_DIMS[1:] for ny in rows_of(P, mgn.ISTA_DIMS[0])]
    CDiag = pm.MPIBlockDiag([pm.local.NonStationaryConvolve1D(d, hs, ih, axis=-1) for d in dims])
    d = CDiag @ pm.DistributedArray.to_dist(m)
    np.testing.assert_allclose(host(d.asarray()), GOLD["ista/d"], rtol=1e-12, atol=1e-12)
    x0 = pm.DistributedArray.to_dist(np.zeros_like(m))
    x, iiter, cost = pm.ista(CDiag, d, x0, niter=mgn.ISTA_NITER, eps=mgn.ISTA_EPS, alpha=alpha, tol=1e-10)
    assert iiter == int(GOLD[f"ista/P{P}/iiter"])
    np.testing.assert_allclose(cost, GOLD[f"ista/P{P}/cost"], rtol=1e-10)
    np.testing.assert_allclose(host(x.asarray()), GOLD[f"ista/P{P}/x"], rtol=1e-9, atol=1e-11)
