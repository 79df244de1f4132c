"""Rank-local Kirchhoff demigration (pylops.waveeqprocessing.Kirchhoff / LSM inside MPIVStack, tutorials/lsm.py).

CPU: refshim's restatement against explicit dense matrices built from the definition, the traveltime tables of
``local`` against the restatement's, and the fixtures of tests/golden/kirchhoff_golden.npz (made by
make_golden_kirchhoff.py: the reference's MPIVStack and cgls over the restatement).  GPU: the b2_kirchhoff kernel
through the C ABI against the vectorised NumPy restatement, and the operators through the public interface."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_kirchhoff as mgk  # noqa: E402
from op_checks import (assert_cgls_replay_matches_steps, assert_rejected, guarded_twice, host,  # noqa: E402
                       needs_gpus, run_on_ranks)

GOLD = np.load(os.path.join(HERE, "golden", "kirchhoff_golden.npz"), allow_pickle=False)
KREF, WAVELETS_MOD = mgk.refshim()
U64, U32 = 2.0 ** -52, 2.0 ** -24
ARG, DT = 2002, 2001
# cgls over 100 iterations magnifies rounding.  The fixture solve was run twice more on the CPU with the sums
# reordered, everything else equal: once with the spreading sums over image points descending, once with both the
# spreading and the stacking sums (over traces) descending.  Over P = 1, 2, 3 the cost history moved by up to 2.1e-2
# (relative) and the model by up to 5.9e-4 of its largest value.  The tolerances are five times that spread.
FLOW_COST_RTOL, FLOW_MINV_ATOL = 0.1, 3e-3


# ---------------------------------------------------------------------------------------------------------------
# the definition as dense matrices
# ---------------------------------------------------------------------------------------------------------------
def spread_matrix(ts, tr, dt, nt):
    """(ns*nr*nt, ni) matrix of the spreading stage, built pair by pair from the definition"""
    ni, ns = ts.shape
    nr = tr.shape[1]
    M = np.zeros((ns * nr * nt, ni))
    for s in range(ns):
        for r in range(nr):
            for ii in range(ni):
                trav = ts[ii, s] + tr[ii, r]
                it = int(trav / dt)
                d = trav / dt - it
                if 0 <= it < nt - 1:
                    row = (s * nr + r) * nt
                    M[row + it, ii] += 1 - d
                    M[row + it + 1, ii] += d
    return M


def conv_matrix(nt, h, off):
    """Convolve1D along one trace: y[i] = sum_k h[k] x[i + off - k]"""
    C = np.zeros((nt, nt))
    for i in range(nt):
        for j in range(nt):
            if 0 <= i + off - j < len(h):
                C[i, j] = h[i + off - j]
    return C


def op_matrix(ts, tr, dt, nt, h, off):
    ntr = ts.shape[1] * tr.shape[1]
    return np.kron(np.eye(ntr), conv_matrix(nt, h, off)) @ spread_matrix(ts, tr, dt, nt)


def small_geometry(nt=14, dt=0.004):
    z, x, t, srcs, recs, vel = mgk.op_geometry(1)
    t = np.arange(nt) * dt
    return z, x, t, srcs, recs, vel


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wav", ["spike", "asym/o0", "asym/o4", "ricker21"])
@pytest.mark.parametrize("nt", [2, 3, 9, 14, 40])
def test_refshim_kirchhoff_is_the_dense_definition(wav, nt):
    z, x, t, srcs, recs, vel = small_geometry(nt)
    h, off = mgk.wavelet(wav)
    Op = KREF.Kirchhoff(z, x, t, srcs, recs, vel, h, off, mode="analytic")
    assert Op.shape == (srcs.shape[1] * recs.shape[1] * nt, x.size * z.size)
    M = op_matrix(Op.trav_srcs, Op.trav_recs, Op.dt, nt, h, off)
    rng = np.random.default_rng(nt)
    m, d = rng.standard_normal(Op.shape[1]), rng.standard_normal(Op.shape[0])
    scale = np.abs(M).sum() + 1
    np.testing.assert_allclose(Op.matvec(m), M @ m, rtol=0, atol=1e-13 * scale)
    np.testing.assert_allclose(Op.rmatvec(d), M.T @ d, rtol=0, atol=1e-13 * scale)


def test_refshim_spread_stack_are_pylops_loops_in_pylops_order():
    """the vectorised stages against the literal loops (same operations, same order): equal bit for bit"""
    z, x, t, srcs, recs, vel = small_geometry(14)
    ts, tr = KREF.traveltime_tables(z, x, srcs, recs, vel)
    ni, ns, nr, nt, dt = ts.shape[0], ts.shape[1], tr.shape[1], 14, 0.004
    rng = np.random.default_rng(2)
    for dtype in (np.float64, np.float32):
        m = rng.standard_normal(ni).astype(dtype)
        d = rng.standard_normal((ns * nr, nt)).astype(dtype)
        yf = np.zeros((ns * nr, nt), dtype)
        ya = np.zeros(ni, dtype)
        for s in range(ns):
            for r in range(nr):
                for ii in range(ni):
                    trav = ts[ii, s] + tr[ii, r]
                    it = int(trav / dt)
                    w = trav / dt - it
                    if 0 <= it < nt - 1:
                        yf[s * nr + r, it] += m[ii] * (1 - w)
                        yf[s * nr + r, it + 1] += m[ii] * w
        for ii in range(ni):
            for s in range(ns):
                for r in range(nr):
                    trav = ts[ii, s] + tr[ii, r]
                    it = int(trav / dt)
                    w = trav / dt - it
                    if 0 <= it < nt - 1:
                        ya[ii] += d[s * nr + r, it] * (1 - w) + d[s * nr + r, it + 1] * w
        np.testing.assert_array_equal(KREF.spread(m, ts, tr, dt, nt, dtype), yf)
        np.testing.assert_array_equal(KREF.stack(d, ts, tr, dt, nt, dtype), ya)


@pytest.mark.parametrize("geom", ["op", "flow"])
def test_local_tables_equal_the_restatement(geom):
    from pylops_mpi_b200.local import _traveltime_tables
    if geom == "op":
        z, x, t, srcs, recs, vel = mgk.op_geometry(3)
    else:
        z, x, t, srcs, recs, vel, *_ = mgk.flow_setup(2, 1)
    a = _traveltime_tables(z, x, srcs, recs, vel)
    b = KREF.traveltime_tables(z, x, srcs, recs, vel)
    for u, v in zip(a, b):
        assert u.dtype == np.float64 and u.shape == v.shape
        np.testing.assert_array_equal(u, v)


def test_ricker_restatement():
    w, tw, wc = WAVELETS_MOD.ricker(np.arange(41) * 0.004, f0=20)
    assert w.size == 81 and tw.size == 81 and wc == 40 and w[40] == 1.0
    np.testing.assert_array_equal(w, w[::-1])
    w2, _, wc2 = WAVELETS_MOD.ricker(np.arange(42) * 0.004, f0=20)        # an even t loses its last sample
    np.testing.assert_array_equal(w2, w)
    assert wc2 == wc


def test_kirchhoff_fixture_inventory():
    names = set()
    for P in (1, 2, 3):
        for wav in mgk.WAVELETS:
            y, ya = GOLD[f"{mgk.key(P, wav)}/y"], GOLD[f"{mgk.key(P, wav)}/ya"]
            assert y.dtype == np.float64 and y.shape == (P * mgk.OP_NS * mgk.OP_NR * mgk.OP_NT,)
            assert ya.dtype == np.float64 and ya.shape == (mgk.OP_NX * mgk.OP_NZ,)
            names |= {f"{mgk.key(P, wav)}/y", f"{mgk.key(P, wav)}/ya"}
        for k in ("madj", "minv", "iiter", "cost"):
            names.add(f"flow/P{P}/{k}")
        assert int(GOLD[f"flow/P{P}/iiter"]) == mgk.FLOW_NITER
        assert GOLD[f"flow/P{P}/cost"].shape == (mgk.FLOW_NITER + 1,)
        assert GOLD[f"flow/P{P}/minv"].shape == GOLD[f"flow/P{P}/madj"].shape == (mgk.FLOW_NX * mgk.FLOW_NZ,)
    assert sorted(GOLD.files) == sorted(names)
    assert os.path.getsize(os.path.join(HERE, "golden", "kirchhoff_golden.npz")) < 400_000


@pytest.mark.parametrize("P", [1, 2, 3])
@pytest.mark.parametrize("wav", mgk.WAVELETS)
def test_kirchhoff_fixtures_follow_the_definition(P, wav):
    z, x, t, srcs, recs, vel = mgk.op_geometry(P)                 # all P ranks' sources: the gathered operator
    ts, tr = KREF.traveltime_tables(z, x, srcs, recs, vel)
    h, off = mgk.wavelet(wav)
    M = op_matrix(ts, tr, mgk.OP_DT, mgk.OP_NT, h, off)
    m, d = mgk.op_inputs(P)
    y, ya = GOLD[f"{mgk.key(P, wav)}/y"], GOLD[f"{mgk.key(P, wav)}/ya"]
    np.testing.assert_allclose(y, M @ m, rtol=0, atol=1e-13 * np.abs(y).max())
    np.testing.assert_allclose(ya, M.T @ d, rtol=0, atol=1e-13 * np.abs(ya).max())


@pytest.mark.parametrize("P", [1, 3])
def test_kirchhoff_flow_fixture_madj_follows_the_restatement(P):
    z, x, t, srcs, recs, v0, wav, wavc, refl = mgk.flow_setup(P)
    Op = KREF.Kirchhoff(z, x, t, srcs, recs, v0, wav, wavc, mode="analytic")
    madj = Op.rmatvec(Op.matvec(refl.ravel()))
    np.testing.assert_allclose(GOLD[f"flow/P{P}/madj"], madj, rtol=0, atol=1e-12 * np.abs(madj).max())


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernel through the C ABI
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


def c_kirch(pm, x, y, ts, tr, ni, ns, nr, nt, dt, adjoint, code):
    L = pm._lib
    return L.lib.b2_kirchhoff(L.ctx(), x, y, ts, tr, ni, ns, nr, nt, dt, adjoint, code, L.stream())


def tables(ni, ns, nr, nt, dt, seed):
    """(ni, ns), (nr, ni) float64 tables whose pairs cover [0, nt + 3) samples: some land past the record, some on
    nt - 2 / nt - 1, and one pair of every trace sits at trav = 0 or on a sample exactly"""
    rng = np.random.default_rng(seed)
    ts = rng.uniform(0, (nt + 3) * dt / 2, (ni, ns))
    tr = rng.uniform(0, (nt + 3) * dt / 2, (ni, nr))
    ts[0], tr[0] = 0.0, 0.0
    ts[1 % ni], tr[1 % ni] = (nt - 2) * dt / 2, (nt - 2) * dt / 2
    return ts, tr


def run_kernel(pm, x_np, ts, tr, nt, dt, adjoint, dtype, guard=3):
    """b2_kirchhoff into an output at an odd element offset inside a guarded buffer; returns (y, guards intact,
    second apply bit-equal)"""
    import torch
    ni, ns = ts.shape
    nr = tr.shape[1]
    x = torch.as_tensor(np.ascontiguousarray(x_np.ravel().astype(dtype))).cuda()
    tsd = torch.as_tensor(np.ascontiguousarray(ts.T)).cuda()
    trd = torch.as_tensor(np.ascontiguousarray(tr.T)).cuda()
    code = pm._lib.F32 if dtype == np.float32 else pm._lib.F64
    args = (tsd.data_ptr(), trd.data_ptr(), ni, ns, nr, nt, dt, int(adjoint), code)
    return guarded_twice(lambda yp: c_kirch(pm, x.data_ptr(), yp, *args), ni if adjoint else ns * nr * nt, dtype,
                         guard, 1)


def forward_bound(x, ts, tr, dt, nt):
    """per sample: the sum of the magnitudes of its contributions, and n, their number"""
    mag = KREF.spread(np.abs(x.astype(np.float64)), ts, tr, dt, nt, np.float64)
    return mag, count_contributions(ts, tr, dt, nt)


def count_contributions(ts, tr, dt, nt):
    ni, ns = ts.shape
    nr = tr.shape[1]
    c = np.zeros((ns * nr) * nt)
    trav = (ts[:, :, None] + tr[:, None, :]).reshape(ni, ns * nr).T
    it, _, ok = KREF.pair_index(trav, dt, nt)
    isr, ii = np.nonzero(ok)
    base = isr * nt + it[isr, ii]
    np.add.at(c, base, 1)
    np.add.at(c, base + 1, 1)
    return c.reshape(ns * nr, nt)


def check_kernel(pm, ni, ns, nr, nt, dt, dtype, seed):
    ts, tr = tables(ni, ns, nr, nt, dt, seed)
    rng = np.random.default_rng(seed + 1)
    m = rng.standard_normal(ni).astype(dtype)
    d = rng.standard_normal(ns * nr * nt).astype(dtype)
    y, guards, same = run_kernel(pm, m, ts, tr, nt, dt, False, dtype)
    assert guards and same
    ref = KREF.spread(m.astype(np.float64), ts, tr, dt, nt, np.float64).ravel()
    mag, n = forward_bound(m, ts, tr, dt, nt)
    u = U64 if dtype == np.float64 else U32
    err = np.abs(y.astype(np.float64) - ref)
    assert np.all(err <= n.ravel() * u * mag.ravel()), f"forward: max err {err.max():.3e}"
    ya, guards, same = run_kernel(pm, d, ts, tr, nt, dt, True, dtype)
    assert guards and same
    refa = KREF.stack(d.reshape(ns * nr, nt).astype(np.float64), ts, tr, dt, nt, np.float64)
    if dtype == np.float64:
        np.testing.assert_array_equal(ya, refa)                      # pylops' order: bit for bit
    else:
        maga = KREF.stack(np.abs(d.reshape(ns * nr, nt).astype(np.float64)), ts, tr, dt, nt, np.float64)
        na = ns * nr * 2
        err = np.abs(ya.astype(np.float64) - refa)
        assert np.all(err <= na * U32 * maga + U32 * np.abs(refa)), f"adjoint: max err {err.max():.3e}"


# nt = 1472 / 1473 (float64) and 2944 / 2945 (float32): the last trace length accumulated in shared memory, and the
# first one accumulated in global memory
SHAPES = [(117, 2, 5, 14), (117, 2, 5, 1), (117, 2, 5, 2), (117, 2, 5, 3), (64, 3, 4, 4), (33, 1, 1, 7),
          (1000, 4, 9, 500), (4860, 10, 11, 651), (77, 3, 2, 1472), (77, 3, 2, 1473), (70, 2, 3, 2944),
          (70, 2, 3, 2945)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"ni{s[0]}-ns{s[1]}-nr{s[2]}-nt{s[3]}" for s in SHAPES])
def test_kernel_vs_numpy(pm, dtype, shape):
    ni, ns, nr, nt = shape
    check_kernel(pm, ni, ns, nr, nt, 0.004, dtype, sum(shape))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_kernel_more_than_65535_traces(pm, dtype):
    check_kernel(pm, 9, 300, 250, 16, 0.002, dtype, 3)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_kernel_trace_beyond_shared_memory(pm, dtype):
    check_kernel(pm, 40, 2, 3, 40000, 0.001, dtype, 4)


@pytest.mark.gpu
def test_kernel_tutorial_tables_adjoint_bitwise(pm):
    """the tutorial's own tables and dt (0.004, whose division is where 1/dt or float32 shortcuts go wrong)"""
    z, x, t, srcs, recs, v0, *_ = mgk.flow_setup(1)
    ts, tr = KREF.traveltime_tables(z, x, srcs, recs, v0)
    nt, dt = t.size, t[1] - t[0]
    d = np.random.default_rng(6).standard_normal(ts.shape[1] * tr.shape[1] * nt)
    ya, guards, same = run_kernel(pm, d, ts, tr, nt, dt, True, np.float64)
    assert guards and same
    np.testing.assert_array_equal(ya, KREF.stack(d.reshape(-1, nt), ts, tr, dt, nt, np.float64))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(117, 2, 5, 14), (1000, 4, 9, 500), (60, 2, 2, 5000)])
def test_kernel_adjoint_dot(pm, shape):
    ni, ns, nr, nt = shape
    ts, tr = tables(ni, ns, nr, nt, 0.004, 9)
    rng = np.random.default_rng(10)
    m, d = rng.standard_normal(ni), rng.standard_normal(ns * nr * nt)
    fm, _, _ = run_kernel(pm, m, ts, tr, nt, 0.004, False, np.float64)
    ad, _, _ = run_kernel(pm, d, ts, tr, nt, 0.004, True, np.float64)
    lhs, rhs = np.dot(fm, d), np.dot(m, ad)
    assert abs(lhs - rhs) <= 1e-12 * np.linalg.norm(fm) * np.linalg.norm(d)


@pytest.mark.gpu
def test_kernel_error_codes_leave_y_untouched(pm):
    import torch
    L = pm._lib
    ni, ns, nr, nt = 6, 2, 3, 5
    x = torch.ones(ns * nr * nt, dtype=torch.float64, device="cuda")
    y = torch.full((ns * nr * nt,), 3.5, dtype=torch.float64, device="cuda")
    ts = torch.zeros(ns * ni, dtype=torch.float64, device="cuda")
    tr = torch.zeros(nr * ni, dtype=torch.float64, device="cuda")
    cases = [
        (dict(x=None), ARG), (dict(y=None), ARG), (dict(ts=None), ARG), (dict(tr=None), ARG), (dict(y="x"), ARG),
        (dict(ni=0), ARG), (dict(ns=0), ARG), (dict(nr=0), ARG), (dict(nt=0), ARG),
        (dict(dt=0.0), ARG), (dict(dt=-0.004), ARG), (dict(dt=float("inf")), ARG), (dict(dt=float("nan")), ARG),
        (dict(dtype=L.C64), DT), (dict(dtype=L.C128), DT), (dict(dtype=L.BF16), DT), (dict(dtype=99), DT),
    ]
    for adjoint in (0, 1):
        assert_rejected(lambda a: L.lib.b2_kirchhoff(a["ctx"], a["x"], a["y"], a["ts"], a["tr"], a["ni"], a["ns"], a["nr"],
                                                     a["nt"], a["dt"], adjoint, a["dtype"], L.stream()),
                        dict(ctx=L.ctx(), x=x.data_ptr(), y=y.data_ptr(), ts=ts.data_ptr(), tr=tr.data_ptr(), ni=ni,
                             ns=ns, nr=nr, nt=nt, dt=0.004, dtype=L.F64), cases + [(dict(ctx=None), ARG)], y)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the operators
# ---------------------------------------------------------------------------------------------------------------
def op_vstack(pm, P, wav, dtype="float64"):
    """the P ranks' operators of an operator case, as one MPIVStack on this GPU"""
    h, off = mgk.wavelet(wav)
    ops = []
    for r in range(P):
        z, x, t, srcs, recs, vel = mgk.op_geometry(P, r)
        ops.append(pm.local.Kirchhoff(z, x, t, srcs, recs, vel, h, off, mode="analytic", dtype=dtype))
    return pm.MPIVStack(ops)


def bcast(pm, a):
    return pm.DistributedArray.to_dist(a, partition=pm.Partition.BROADCAST)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
@pytest.mark.parametrize("wav", mgk.WAVELETS)
def test_operator_vs_reference_fixtures(pm, P, wav):
    Op = op_vstack(pm, P, wav)
    m, d = mgk.op_inputs(P)
    y = host((Op @ bcast(pm, m)).asarray())
    ya = host((Op.H @ pm.DistributedArray.to_dist(d)).asarray())
    gy, gya = GOLD[f"{mgk.key(P, wav)}/y"], GOLD[f"{mgk.key(P, wav)}/ya"]
    np.testing.assert_allclose(y, gy, rtol=0, atol=1e-12 * np.abs(gy).max())
    if wav == "spike" and P == 1:
        np.testing.assert_array_equal(ya, gya)            # identity convolution, one rank: pylops' stacking exactly
    else:
        np.testing.assert_allclose(ya, gya, rtol=0, atol=1e-12 * np.abs(gya).max())
    # float32 operator: 100 float32 ulps of the largest value
    Op32 = op_vstack(pm, P, wav, "float32")
    y32 = host((Op32 @ bcast(pm, m.astype(np.float32))).asarray())
    ya32 = host((Op32.H @ pm.DistributedArray.to_dist(d.astype(np.float32))).asarray())
    assert y32.dtype == np.float32 and ya32.dtype == np.float32
    np.testing.assert_allclose(y32, gy, rtol=0, atol=100 * U32 * np.abs(gy).max())
    np.testing.assert_allclose(ya32, gya, rtol=0, atol=100 * U32 * np.abs(gya).max())


@pytest.mark.gpu
def test_single_operator_spike_adjoint_bitwise_every_rank(pm):
    """each rank's operator alone (no all-reduce): the f64 adjoint with the identity wavelet is pylops' loop exactly"""
    import torch
    for P in (2, 3):
        m, d = mgk.op_inputs(P)
        n = mgk.OP_NS * mgk.OP_NR * mgk.OP_NT
        for r in range(P):
            z, x, t, srcs, recs, vel = mgk.op_geometry(P, r)
            K = pm.local.Kirchhoff(z, x, t, srcs, recs, vel, [1.0], 0, mode="analytic")
            ts, tr = KREF.traveltime_tables(z, x, srcs, recs, vel)
            got = host(K.rmatvec(torch.as_tensor(d[r * n:(r + 1) * n]).cuda()))
            np.testing.assert_array_equal(got, KREF.stack(d[r * n:(r + 1) * n], ts, tr, mgk.OP_DT, mgk.OP_NT,
                                                          np.float64))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_operator_dottest(pm, dtype):
    Op = op_vstack(pm, 2, "ricker21", dtype)
    rng = np.random.default_rng(5)
    u = bcast(pm, rng.standard_normal(Op.shape[1]).astype(dtype))
    v = pm.DistributedArray.to_dist(rng.standard_normal(Op.shape[0]).astype(dtype))
    assert pm.dottest(Op, u, v, rtol=1e-4 if dtype == "float32" else 1e-12)


@pytest.mark.gpu
def test_operator_complex_data_and_out(pm):
    import torch
    z, x, t, srcs, recs, vel = mgk.op_geometry(1)
    h, off = mgk.wavelet("asym/o4")
    K = pm.local.Kirchhoff(z, x, t, srcs, recs, vel, h, off, mode="analytic")
    assert K.shape == (mgk.OP_NS * mgk.OP_NR * mgk.OP_NT, mgk.OP_NX * mgk.OP_NZ)
    assert K.dims == (mgk.OP_NX, mgk.OP_NZ) and K.dimsd == (mgk.OP_NS, mgk.OP_NR, mgk.OP_NT)
    rng = np.random.default_rng(7)
    for adjoint in (False, True):
        n = K.shape[0] if adjoint else K.shape[1]
        a = torch.as_tensor(rng.standard_normal(n) + 1j * rng.standard_normal(n)).cuda()
        f = K.rmatvec if adjoint else K.matvec
        y = f(a)
        assert y.dtype == torch.complex128


@pytest.mark.gpu
def test_operator_argument_errors(pm):
    z, x, t, srcs, recs, vel = mgk.op_geometry(1)
    h = np.ones(3)
    K = pm.local.Kirchhoff
    for kw, name in ((dict(mode="eikonal"), "mode"), (dict(mode="byot"), "mode"), (dict(dynamic=True), "dynamic"),
                     (dict(wavfilter=True), "wavfilter"), (dict(trav=np.zeros((2, 2))), "trav"),
                     (dict(amp=np.zeros((2, 2))), "amp"), (dict(aperture=2.0), "aperture"),
                     (dict(angleaperture=45), "angleaperture"), (dict(snell=30.0), "snell"),
                     (dict(y=np.arange(3.0)), "y")):
        kw = {"mode": "analytic", **kw}
        with pytest.raises(NotImplementedError, match=name):
            K(z, x, t, srcs, recs, vel, h, 1, **kw)
    with pytest.raises(NotImplementedError, match="mode"):
        K(z, x, t, srcs, recs, vel, h, 1)                                   # pylops' default mode is eikonal
    with pytest.raises(ValueError):
        K(z, x, t, srcs, recs, np.full((x.size, z.size), 1000.0), h, 1, mode="analytic")
    assert K(z, x, t, srcs, recs, vel, h, 1, mode="analytic", engine="numba").engine == "numba"
    with pytest.raises(NotImplementedError):
        pm.local.LSM(z, x, t, srcs, recs, vel, h, 1, kind="wave", mode="analytic")
    with pytest.raises(NotImplementedError):
        pm.local.LSM(z, x, t, srcs, recs, vel, h, 1, dottest=True, mode="analytic")
    lsm = pm.local.LSM(z, x, t, srcs, recs, vel, h, 1, mode="analytic", dtype="float32")
    assert type(lsm.Demop).__name__ == "Kirchhoff" and lsm.Demop.dtype == np.float32


def check_flow(P, madj, minv, iiter, cost):
    g = f"flow/P{P}"
    gm = GOLD[f"{g}/madj"]
    np.testing.assert_allclose(madj, gm, rtol=0, atol=1e-12 * np.abs(gm).max())
    assert int(iiter) == int(GOLD[f"{g}/iiter"])
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"{g}/cost"], rtol=FLOW_COST_RTOL)
    gi = GOLD[f"{g}/minv"]
    np.testing.assert_allclose(minv, gi, rtol=0, atol=FLOW_MINV_ATOL * np.abs(gi).max())


@pytest.mark.gpu
def test_tutorial_lsm_line_for_line(pm):
    """tutorials/lsm.py on one rank, statement by statement, with pylops_mpi_b200 in place of pylops_mpi and
    local.LSM in place of pylops.waveeqprocessing.lsm.LSM"""
    import pylops_mpi_b200 as pylops_mpi
    from pylops_mpi_b200.local import LSM
    ricker = WAVELETS_MOD.ricker
    rank, size = 0, 1

    nx, nz = 81, 60
    dx, dz = 4, 4
    x, z = np.arange(nx) * dx, np.arange(nz) * dz
    v0 = 1000
    refl = np.zeros((nx, nz))
    refl[:, 30] = -1
    refl[:, 50] = 0.5
    nr = 11
    rx = np.linspace(10 * dx, (nx - 10) * dx, nr)
    rz = 20 * np.ones(nr)
    recs = np.vstack((rx, rz))
    ns = 10
    nstot = ns * size
    sxtot = np.linspace(dx * 10, (nx - 10) * dx, nstot)
    sx = sxtot[rank * ns: (rank + 1) * ns]
    sz = 10 * np.ones(ns)
    sources = np.vstack((sx, sz))

    nt = 651
    dt = 0.004
    t = np.arange(nt) * dt
    wav, wavt, wavc = ricker(t[:41], f0=20)

    lsm = LSM(z, x, t, sources, recs, v0, wav, wavc, mode="analytic", engine="numba")

    VStack = pylops_mpi.MPIVStack(ops=[lsm.Demop, ])
    refl_dist = pylops_mpi.DistributedArray(global_shape=nx * nz, partition=pylops_mpi.Partition.BROADCAST)
    refl_dist[:] = refl.flatten()
    d_dist = VStack @ refl_dist
    d = d_dist.asarray().reshape((nstot, nr, nt))

    madj_dist = VStack.H @ d_dist
    madj = madj_dist.asarray().reshape((nx, nz))
    d_adj_dist = VStack @ madj_dist
    d_adj = d_adj_dist.asarray().reshape((nstot, nr, nt))

    x0 = pylops_mpi.DistributedArray(VStack.shape[1], partition=pylops_mpi.Partition.BROADCAST)
    x0[:] = 0
    minv_dist, _, iiter, _, _, cost = pylops_mpi.cgls(VStack, d_dist, x0=x0, niter=100, show=False)
    minv = minv_dist.asarray().reshape((nx, nz))
    d_inv_dist = VStack @ minv_dist
    d_inv = d_inv_dist.asarray().reshape(nstot, nr, nt)

    check_flow(1, host(madj).ravel(), host(minv).ravel(), iiter, cost)
    Kr = KREF.Kirchhoff(z, x, t, sources, recs, v0, wav, wavc, mode="analytic")
    dref = Kr.matvec(refl.ravel())
    np.testing.assert_allclose(host(d).ravel(), dref, rtol=0, atol=1e-12 * np.abs(dref).max())
    assert d_adj.shape == d_inv.shape == (nstot, nr, nt)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
def test_tutorial_flow_vs_reference(pm, P):
    """the tutorial's flow with the sources of P ranks held as P operators of one MPIVStack; cgls replays its graph"""
    from pylops_mpi_b200.optimization.cls_basic import _graph_safe
    ops = []
    for r in range(P):
        z, x, t, srcs, recs, v0, wav, wavc, refl = mgk.flow_setup(P, r)
        ops.append(pm.local.LSM(z, x, t, srcs, recs, v0, wav, wavc, mode="analytic").Demop)
    VStack = pm.MPIVStack(ops)
    assert _graph_safe(VStack)
    d = VStack @ bcast(pm, refl.ravel())
    madj = VStack.H @ d
    x0 = bcast(pm, np.zeros(VStack.shape[1]))
    minv, _, iiter, _, _, cost = pm.cgls(VStack, d, x0=x0, niter=mgk.FLOW_NITER)
    check_flow(P, host(madj.asarray()), host(minv.asarray()), iiter, cost)


@pytest.mark.gpu
def test_cgls_graph_replay_matches_step_loop(pm):
    Op = op_vstack(pm, 2, "ricker21")
    rng = np.random.default_rng(12)
    y = Op @ bcast(pm, rng.standard_normal(Op.shape[1]))
    assert_cgls_replay_matches_steps(pm, Op, y, bcast(pm, np.zeros(Op.shape[1])), 25, 20)


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [1, 2])
def test_multi_rank_fixtures(nproc):
    needs_gpus(nproc)
    run_on_ranks("test_kirchhoff", nproc)


def on_ranks(pm, comm):
    """each rank's MPIVStack([Kirchhoff]) against its slice of the gathered fixtures, and the LSM flow against its
    fixture"""
    rank, P = comm.Get_rank(), comm.Get_size()

    def close(name, got, ref, atol_rel):
        np.testing.assert_allclose(got, ref, rtol=0, atol=atol_rel * np.abs(ref).max(), err_msg=f"[rank {rank}] {name}")

    n = mgk.OP_NS * mgk.OP_NR * mgk.OP_NT
    ls = [(n,)] * P
    for wav in mgk.WAVELETS:
        h, off = mgk.wavelet(wav)
        z, x, t, srcs, recs, vel = mgk.op_geometry(P, rank)
        Op = pm.MPIVStack([pm.local.Kirchhoff(z, x, t, srcs, recs, vel, h, off, mode="analytic")])
        m, d = mgk.op_inputs(P)
        y = Op @ pm.DistributedArray.to_dist(m, partition=pm.Partition.BROADCAST)
        ya = Op.H @ pm.DistributedArray.to_dist(d, local_shapes=ls)
        k = mgk.key(P, wav)
        close(f"{k}/y", host(y.local_array), GOLD[f"{k}/y"][rank * n:(rank + 1) * n], 1e-12)
        close(f"{k}/ya", host(ya.local_array), GOLD[f"{k}/ya"], 1e-12)

    z, x, t, srcs, recs, v0, wav, wavc, refl = mgk.flow_setup(P, rank)
    lsm = pm.local.LSM(z, x, t, srcs, recs, v0, wav, wavc, mode="analytic", engine="numba")
    VStack = pm.MPIVStack(ops=[lsm.Demop, ])
    refl_dist = pm.DistributedArray(global_shape=refl.size, partition=pm.Partition.BROADCAST)
    refl_dist[:] = refl.flatten()
    d_dist = VStack @ refl_dist
    madj = VStack.H @ d_dist
    x0 = pm.DistributedArray(VStack.shape[1], partition=pm.Partition.BROADCAST)
    x0[:] = 0
    minv, _, iiter, _, _, cost = pm.cgls(VStack, d_dist, x0=x0, niter=mgk.FLOW_NITER)
    g = f"flow/P{P}"
    close(f"{g}/madj", host(madj.local_array), GOLD[f"{g}/madj"], 1e-12)
    assert int(iiter) == int(GOLD[f"{g}/iiter"])
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"{g}/cost"], rtol=FLOW_COST_RTOL, err_msg=f"[rank {rank}] cost")
    close(f"{g}/minv", host(minv.local_array), GOLD[f"{g}/minv"], FLOW_MINV_ATOL)
