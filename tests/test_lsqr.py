"""LSQR: the scalar recurrence (b2_lsqr_scalars) against its float64 NumPy statement, the fused update
(b2_lsqr_update) against float64 references, the solver against scipy.sparse.linalg.lsqr's fixtures
(tests/golden/make_golden_lsqr.py), every mode of running the one device iteration, and LSM.solve."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_lsqr as mgl  # noqa: E402
import make_golden_kirchhoff as mgk  # noqa: E402
from op_checks import host, needs_gpus, run_on_ranks  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "lsqr_golden.npz"), allow_pickle=False)
H = mgl.lsqr_host()
DENSE = ("consistent", "inconsistent", "illcond", "limit", "damped", "x0", "novar", "complex", "float32")
SCALARS = ("r1norm", "r2norm", "anorm", "acond", "arnorm", "xnorm")


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
def test_fixture_inventory():
    expect = {"consistent": 1, "inconsistent": 2, "illcond": 3, "limit": 7, "float32": 7}
    for name in DENSE:
        assert GOLD[f"{name}/cost"].shape == (int(GOLD[f"{name}/itn"]) + 1,)
        assert GOLD[f"{name}/x"].shape == GOLD[f"{name}/var"].shape == (GOLD[f"{name}/A"].shape[1],)
        assert GOLD[f"{name}/spread"].shape == (9,)
        if name in expect:
            assert int(GOLD[f"{name}/istop"]) == expect[name]
    assert GOLD["complex/A"].dtype == np.complex128 and GOLD["complex/var"].dtype == np.complex128
    assert GOLD["float32/A"].dtype == np.float32
    assert not GOLD["novar/var"].any() and GOLD["damped/params"][0] > 0 and GOLD["x0/x0"].any()
    for name in ("flow", "lsm"):
        assert int(GOLD[f"{name}/itn"]) == mgl.FLOW_NITER and 0 < float(GOLD[f"{name}/spread"]) < 1e-2


@pytest.mark.parametrize("name", ["inconsistent", "illcond", "damped", "complex"])
def test_transcription_equals_scipy(name):
    """lsqr_host, driven by scipy's vectors and reductions, reproduces scipy's outputs bit for bit"""
    from scipy.sparse.linalg import lsqr
    A, b = GOLD[f"{name}/A"], GOLD[f"{name}/b"]
    damp, atol, btol, conlim, niter, calc_var, has_x0 = GOLD[f"{name}/params"]
    x0 = GOLD[f"{name}/x0"] if has_x0 else None
    ref = lsqr(A, b, damp=damp, atol=atol, btol=btol, conlim=conlim, iter_lim=int(niter), calc_var=bool(calc_var),
               x0=x0)
    got, _ = mgl.transcription(A, b, damp, atol, btol, conlim, int(niter), bool(calc_var), x0)
    for g, r in zip(got, ref):
        np.testing.assert_array_equal(np.asarray(g), np.asarray(r))


# ---------------------------------------------------------------------------------------------------------------
# GPU: kernels
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


def initial_state(alfa, beta, damp, niter, bnorm):
    s = np.zeros(H._NSTATE)
    s[[H._ALFA, H._BETA, H._RHOBAR, H._PHIBAR, H._CS2, H._INV_ALFA]] = alfa, beta, alfa, beta, -1.0, 1 / alfa
    s[[H._DAMP, H._DAMPSQ, H._ATOL, H._BTOL, H._CTOL, H._BNORM, H._ITER_LIM]] = damp, damp * damp, mgl.ATOL, \
        mgl.BTOL, 1 / mgl.CONLIM, bnorm, niter
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("damp", [0.0, 0.35])
def test_scalars_kernel_bit_equal_to_numpy(pm, damp):
    """phases 0 / 1 / 2 over a sequence of reductions recorded from a scipy-driven run: every state slot and every
    history row equal the NumPy statement bit for bit"""
    import torch
    L = pm._lib
    A, b = GOLD["inconsistent/A"], GOLD["inconsistent/b"]
    n = 40
    # the initial state and the reductions of the scipy-driven run (|u'|^2, |v'|^2, |dk|^2 per iteration)
    seq, init = [], []

    class Rec:
        shape = A.shape

        def matvec(self, v):
            return A @ v

        def rmatvec(self, u):
            return A.T @ u
    orig = H.lsqr_scalars_host

    def spy(st, phase):
        if not init:
            init.append(st.copy())
        if phase == 0:
            seq.append([st[H._BB], 0.0, 0.0])
        else:
            seq[-1][phase] = st[H._AA] if phase == 1 else st[H._DD]
        return orig(st, phase)
    H.lsqr_scalars_host = spy
    try:
        mgl.transcription(Rec(), b, damp, mgl.ATOL, mgl.BTOL, mgl.CONLIM, n, True, None)
    finally:
        H.lsqr_scalars_host = orig
    s = init[0]
    s[H._BB] = 0.0
    dev = torch.from_numpy(s.copy()).cuda()
    hist = torch.full((n, H._NHIST), -7.0, dtype=torch.float64, device="cuda")
    rows = []
    for k, (bb, aa, dd) in enumerate(seq):
        for phase, slot, val in ((0, H._BB, bb), (1, H._AA, aa)):
            s[slot] = val
            dev[slot] = val
            r = H.lsqr_scalars_host(s, phase)
            if r is not None:
                rows.append(r)
            assert L.lib.b2_lsqr_scalars(dev.data_ptr(), phase, hist.data_ptr(), n, L.stream()) == 0
            np.testing.assert_array_equal(host(dev), s, err_msg=f"iteration {k} phase {phase}")
        s[H._DD] = dd              # finished by the next phase 0 (or the phase 2 below)
        dev[H._DD] = dd
    r = H.lsqr_scalars_host(s, 2)
    if r is not None:
        rows.append(r)
    assert L.lib.b2_lsqr_scalars(dev.data_ptr(), 2, hist.data_ptr(), n, L.stream()) == 0
    np.testing.assert_array_equal(host(dev), s)
    h = host(hist)
    assert len(rows) == len(seq) == n
    np.testing.assert_array_equal(h[:len(rows)], np.array(rows))
    assert (h[len(rows):] == -7.0).all()                       # no row past the last finished iteration


@pytest.mark.gpu
def test_scalars_kernel_stop_flag_and_errors(pm):
    import torch
    L = pm._lib
    s = initial_state(1.0, 1.0, 0.0, 5, 1.0)
    s[H._STOPPED] = 1.0
    dev = torch.from_numpy(s).cuda()
    hist = torch.full((5, H._NHIST), -7.0, dtype=torch.float64, device="cuda")
    for phase in (0, 1, 2):
        assert L.lib.b2_lsqr_scalars(dev.data_ptr(), phase, hist.data_ptr(), 5, L.stream()) == 0
    np.testing.assert_array_equal(host(dev), s)
    assert (host(hist) == -7.0).all()
    ARG = 2002
    assert L.lib.b2_lsqr_scalars(None, 0, hist.data_ptr(), 5, L.stream()) == ARG
    assert L.lib.b2_lsqr_scalars(dev.data_ptr(), 3, hist.data_ptr(), 5, L.stream()) == ARG
    assert L.lib.b2_lsqr_scalars(dev.data_ptr(), -1, hist.data_ptr(), 5, L.stream()) == ARG
    assert L.lib.b2_lsqr_scalars(dev.data_ptr(), 0, None, 5, L.stream()) == ARG


def update_reference(x, w, v, var, t1, t2, ir, ia, dt):
    """the kernel's operations in NumPy, each rounded in the data's real type (float32 ops are correctly rounded)"""
    rt = np.float32 if dt in (np.float32, np.complex64) else np.float64
    cx = np.dtype(dt).kind == "c"
    xr, wr, vr = (a.view(rt).copy() for a in (x, w, v))
    T1, T2, IR, IA = (rt(c) for c in (t1, t2, ir, ia))
    dk = IR * wr
    xr = xr + T1 * wr
    wn = IA * vr + T2 * wr
    dd = float(np.sum(dk.astype(np.float64) ** 2))
    out_var = None
    if var is not None:
        vv = var.view(rt).copy()
        if cx:
            dr, di = dk[0::2], dk[1::2]
            vv[0::2] = vv[0::2] + (dr * dr - di * di)
            vv[1::2] = vv[1::2] + (dr * di + di * dr)
        else:
            vv = vv + dk * dk
        out_var = vv.view(dt)
    return xr.view(dt), wn.view(dt), out_var, dd


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.complex64, np.complex128])
@pytest.mark.parametrize("n,off", [(1, 0), (3, 0), (7, 1), (1000, 0), (4097, 1), (300001, 0), (5, 3), (1003, 3),
                                   (300002, 3)])
@pytest.mark.parametrize("calc_var", [True, False])
def test_update_kernel_against_reference(pm, dtype, n, off, calc_var):
    """x, w, var equal the per-operation NumPy reference bit for bit; dd is a float64 sum in another order: its
    relative error is bounded by n * 2^-53 (sum of non-negative terms), checked at 1e-12 for n <= 3e5"""
    import torch
    L = pm._lib
    rng = np.random.default_rng(n + off)
    tdt = pm._lib.torch_dtype(dtype)

    def rnd():
        a = rng.standard_normal(n)
        return (a + 1j * rng.standard_normal(n) if np.dtype(dtype).kind == "c" else a).astype(dtype)
    x, w, v, var = rnd(), rnd(), rnd(), rnd()
    t1, t2, ir, ia = 0.37, -0.81, 1.9, 0.66
    coef = torch.zeros(8, dtype=torch.float64, device="cuda")
    coef[:4] = torch.tensor([t1, t2, ir, ia], dtype=torch.float64)
    bufs = []
    # sentinels before and after; views start at element off + 1 (16-byte aligned: off = 3 for 4-byte reals, off = 1
    # for 8-byte ones, any off for complex128), so every dtype runs both the vector path with its tail and the
    # scalar path
    for a in (x, w, v, var):
        t = torch.full((n + off + 2,), 5.0, dtype=tdt, device="cuda")
        t[off + 1:off + 1 + n] = torch.from_numpy(a).cuda()
        bufs.append(t)
    views = [t[off + 1:off + 1 + n] for t in bufs]
    rc = L.lib.b2_lsqr_update(L.ctx(), views[0].data_ptr(), views[1].data_ptr(), views[2].data_ptr(),
                              views[3].data_ptr() if calc_var else None, n, L.code(tdt), coef.data_ptr(), None,
                              coef.data_ptr() + 8 * 6, L.stream())
    assert rc == 0
    xr, wr, varr, dd = update_reference(x, w, v, var if calc_var else None, t1, t2, ir, ia, dtype)
    np.testing.assert_array_equal(host(views[0]), xr)
    np.testing.assert_array_equal(host(views[1]), wr)
    np.testing.assert_array_equal(host(views[2]), v)
    np.testing.assert_array_equal(host(views[3]), varr if calc_var else var)
    assert abs(float(coef[6]) - dd) <= 1e-12 * dd
    for t in bufs:
        assert host(t[:off + 1]).tolist() == [5.0] * (off + 1) and host(t[off + 1 + n:]).tolist() == [5.0]


@pytest.mark.gpu
def test_update_kernel_stop_flag_and_errors(pm):
    import torch
    L = pm._lib
    n = 64
    x, w, v, var = (torch.ones(n, dtype=torch.float64, device="cuda") for _ in range(4))
    coef = torch.tensor([1.0, 1.0, 1.0, 1.0, 1.0, 7.0], dtype=torch.float64, device="cuda")   # [4]: stop, [5]: dd
    p = [t.data_ptr() for t in (x, w, v, var)]
    dd = coef.data_ptr() + 40
    assert L.lib.b2_lsqr_update(L.ctx(), *p, n, L.F64, coef.data_ptr(), coef.data_ptr() + 32, dd, L.stream()) == 0
    assert host(x).tolist() == [1.0] * n and host(w).tolist() == [1.0] * n and float(coef[5]) == 7.0
    ARG, DT = 2002, 2001
    assert L.lib.b2_lsqr_update(L.ctx(), *p, n, L.BF16, coef.data_ptr(), None, dd, L.stream()) == DT
    assert L.lib.b2_lsqr_update(None, *p, n, L.F64, coef.data_ptr(), None, dd, L.stream()) == ARG
    assert L.lib.b2_lsqr_update(L.ctx(), *p, n, L.F64, None, None, dd, L.stream()) == ARG
    assert L.lib.b2_lsqr_update(L.ctx(), *p, n, L.F64, coef.data_ptr(), None, None, L.stream()) == ARG
    assert L.lib.b2_lsqr_update(L.ctx(), p[0], p[0], p[2], p[3], n, L.F64, coef.data_ptr(), None, dd,
                                L.stream()) == ARG
    assert L.lib.b2_lsqr_update(L.ctx(), p[0], p[1], p[2], p[0], n, L.F64, coef.data_ptr(), None, dd,
                                L.stream()) == ARG
    assert L.lib.b2_lsqr_update(L.ctx(), None, p[1], p[2], p[3], n, L.F64, coef.data_ptr(), None, dd,
                                L.stream()) == ARG
    # n == 0: the rank's |dk|^2 is 0
    assert L.lib.b2_lsqr_update(L.ctx(), None, None, None, None, 0, L.F64, coef.data_ptr(), None, dd,
                                L.stream()) == 0
    assert float(coef[5]) == 0.0
    assert host(x).tolist() == [1.0] * n


# ---------------------------------------------------------------------------------------------------------------
# GPU: the solver
# ---------------------------------------------------------------------------------------------------------------
def blockdiag_problem(pm, name):
    """fixture case `name` as MPIBlockDiag of NBLK MatrixMult blocks, with y and x0 as DistributedArrays"""
    A, b, x0 = GOLD[f"{name}/A"], GOLD[f"{name}/b"], GOLD[f"{name}/x0"]
    m, n = A.shape[0] // mgl.NBLK, A.shape[1] // mgl.NBLK
    Op = pm.MPIBlockDiag([pm.MatrixMult(np.ascontiguousarray(A[i * m:(i + 1) * m, i * n:(i + 1) * n]))
                          for i in range(mgl.NBLK)])
    return Op, pm.DistributedArray.to_dist(b), pm.DistributedArray.to_dist(x0)


def params(name):
    damp, atol, btol, conlim, niter, calc_var, has_x0 = GOLD[f"{name}/params"]
    return dict(damp=float(damp), atol=float(atol), btol=float(btol), conlim=float(conlim), niter=int(niter),
                calc_var=bool(calc_var)), bool(has_x0)


# Tolerances against scipy.  The device runs scipy's recurrence with other roundings: u, v unnormalised (one
# rounding moved per combination), float64 sums in another order, and the operator's own sum order.  LSQR, like every
# Lanczos-type process without reorthogonalisation, amplifies such differences as it converges, so eps does not bound
# them.  The fixture's `spread` measures the amplification on scipy's own loop: every iteration's two vector
# combinations jittered by 4 ulps per component (three seeds; float32 data also scipy run in float32), each quantity
# on the scale it is resolved to -- x and var to their largest entry, r1norm, r2norm and the cost history to the
# initial residual norm cost[0], arnorm = |A^H r| to anorm * cost[0], anorm, acond and xnorm to themselves.  The
# device's per-component differences are roundings of at most a few ulps per vector operation, the size of the
# jitter, so its distance from scipy is of the order of the spread; TOL_FACTOR = 5 (the factor the Kirchhoff flow
# tolerances put on their rerun spreads) allows for the maximum over three seeds understating the spread, with a
# floor of 100 eps of the data's type.
TOL_FACTOR = 5.0


def tol(name, k):
    eps = np.finfo(np.float32 if name == "float32" else np.float64).eps
    return max(TOL_FACTOR * float(GOLD[f"{name}/spread"][k]), 100 * eps)


def scalar_scale(name, k):
    """the scale spread_of (make_golden_lsqr.py) resolves scalar k to"""
    c0 = float(GOLD[f"{name}/cost"][0])
    return {"r1norm": c0, "r2norm": c0, "arnorm": float(GOLD[f"{name}/anorm"]) * c0}.get(k, abs(float(GOLD[f"{name}/{k}"])))


@pytest.mark.gpu
@pytest.mark.parametrize("name", DENSE)
def test_lsqr_matches_scipy_fixture(pm, name):
    kw, has_x0 = params(name)
    Op, y, x0 = blockdiag_problem(pm, name)
    x, istop, itn, r1, r2, anorm, acond, arnorm, xnorm, var, cost = pm.lsqr(Op, y, x0=x0 if has_x0 else None, **kw)
    assert istop == int(GOLD[f"{name}/istop"]) and itn == int(GOLD[f"{name}/itn"])
    xg = GOLD[f"{name}/x"]
    np.testing.assert_allclose(host(x.asarray()), xg, rtol=0, atol=tol(name, 0) * np.abs(xg).max())
    vg = GOLD[f"{name}/var"]
    np.testing.assert_allclose(host(var.asarray()), vg, rtol=0, atol=tol(name, 1) * max(np.abs(vg).max(), 1e-300))
    for i, (k, got) in enumerate(zip(SCALARS, (r1, r2, anorm, acond, arnorm, xnorm))):
        ref = float(GOLD[f"{name}/{k}"])
        assert abs(got - ref) <= tol(name, 2 + i) * scalar_scale(name, k), (k, got, ref)
    cg = GOLD[f"{name}/cost"]
    np.testing.assert_allclose(cost, cg, rtol=0, atol=tol(name, 8) * cg[0])
    assert var.dtype == x.dtype


MODES = ("graph", "eager", "step", "show", "callback")


def run_mode(pm, Op, Eop, y, x0, kw, mode):
    from pylops_mpi_b200.optimization.cls_basic import LSQR
    s = LSQR(Eop if mode == "eager" else Op)
    if mode == "callback":
        s.callback = lambda x: None
    if mode == "step":
        x = s.setup(y=y, x0=x0, **kw)
        while s.iiter < kw["niter"] and s.istop == 0:
            x = s.step(x)
        s.finalize()
        out = (x, s.istop, s.iiter, s.r1norm, s.r2norm, s.anorm, s.acond, s.arnorm, s.xnorm, s.var, s.cost)
    else:
        out = s.solve(y, x0, show=mode == "show", **kw)
    return s, [host(o.asarray()) if hasattr(o, "asarray") else np.asarray(o) for o in out]


def delegate(pm, blocks):
    from pylops_mpi_b200.local import LocalOperator

    class Delegate(LocalOperator):
        def __init__(self, op):
            self.op, self.shape, self.dtype = op, op.shape, op.dtype

        def _matvec(self, x):
            return self.op.matvec(x)

        def _rmatvec(self, x):
            return self.op.rmatvec(x)
    return [Delegate(b) for b in blocks]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["consistent", "illcond", "damped", "complex", "float32"])
@pytest.mark.parametrize("layout", ["blockdiag", "vstack"])
def test_lsqr_modes_give_identical_bits(pm, capsys, name, layout):
    """graph replay, eager run() (operator off the graph-safe list), a step() loop, show=True and a callback all
    run the one body: identical bits in x, var, every scalar and the cost, including stops inside a block"""
    kw, has_x0 = params(name)
    A, b = GOLD[f"{name}/A"], GOLD[f"{name}/b"]
    m, n = A.shape[0] // mgl.NBLK, A.shape[1] // mgl.NBLK
    if layout == "blockdiag":
        blocks = [pm.MatrixMult(np.ascontiguousarray(A[i * m:(i + 1) * m, i * n:(i + 1) * n])) for i in range(mgl.NBLK)]
        Op, Eop = pm.MPIBlockDiag(blocks), pm.MPIBlockDiag(delegate(pm, blocks))
        y, x0 = pm.DistributedArray.to_dist(b), pm.DistributedArray.to_dist(GOLD[f"{name}/x0"])
    else:                                       # BROADCAST model: the unfused v-step and the share-only |dk|^2
        blocks = [pm.MatrixMult(np.ascontiguousarray(A[i * m:(i + 1) * m, :n])) for i in range(mgl.NBLK)]
        Op, Eop = pm.MPIVStack(blocks), pm.MPIVStack(delegate(pm, blocks))
        y = pm.DistributedArray.to_dist(b)
        x0 = pm.DistributedArray.to_dist(GOLD[f"{name}/x0"][:n], partition=pm.Partition.BROADCAST)
    x0 = x0 if has_x0 else None
    s, ref = run_mode(pm, Op, Eop, y, x0, kw, "graph")
    assert s.graph_error is None and s.graph_replays > 0, s.graph_error
    for mode in MODES[1:]:
        s, got = run_mode(pm, Op, Eop, y, x0, kw, mode)
        if mode == "eager":
            assert s.graph_replays == 0 and s.graph_error == "operator not on the graph-safe list"
        for i, (g, r) in enumerate(zip(got, ref)):
            np.testing.assert_array_equal(g, r, err_msg=f"{mode}: output {i}")
    assert "r2norm" in capsys.readouterr().out


@pytest.mark.gpu
def test_lsqr_callback_sees_every_iteration(pm):
    from pylops_mpi_b200.optimization.cls_basic import LSQR
    Op, y, _ = blockdiag_problem(pm, "limit")
    seen = []
    x, istop, itn, *_ = pm.lsqr(Op, y, niter=12, callback=lambda x: seen.append(host(x.asarray())))
    assert itn == 12 and len(seen) == 12
    s = LSQR(Op)
    xs = s.setup(y=y, niter=12)
    for got in seen:
        xs = s.step(xs)
        np.testing.assert_array_equal(got, host(xs.asarray()))


@pytest.mark.gpu
def test_lsqr_stacked_generic_path(pm):
    """StackedDistributedArray data take the generic path (reference-style operations, host scalars through
    lsqr_host): same fixture, same tolerances as the fused path"""
    from pylops_mpi_b200.optimization.cls_basic import LSQR
    name = "inconsistent"
    kw, _ = params(name)
    A, b = GOLD[f"{name}/A"], GOLD[f"{name}/b"]
    m, n = A.shape[0] // mgl.NBLK, A.shape[1] // mgl.NBLK
    ops = [pm.MPIBlockDiag([pm.MatrixMult(np.ascontiguousarray(A[i * m:(i + 1) * m, i * n:(i + 1) * n]))])
           for i in range(mgl.NBLK)]
    Op = pm.MPIStackedBlockDiag(ops)
    y = pm.StackedDistributedArray([pm.DistributedArray.to_dist(b[i * m:(i + 1) * m]) for i in range(mgl.NBLK)])
    s = LSQR(Op)
    x, istop, itn, r1, *_ , cost = s.solve(y, None, **kw)
    assert s._gen
    assert istop == int(GOLD[f"{name}/istop"]) and itn == int(GOLD[f"{name}/itn"])
    xg = GOLD[f"{name}/x"]
    got = np.concatenate([host(d.asarray()) for d in x.distarrays])
    np.testing.assert_allclose(got, xg, rtol=0, atol=tol(name, 0) * np.abs(xg).max())
    cg = GOLD[f"{name}/cost"]
    np.testing.assert_allclose(cost, cg, rtol=0, atol=tol(name, 8) * cg[0])


def flow_ops(pm, P, rank):
    ops = []
    for r in ([rank] if rank is not None else range(P)):
        z, x, t, srcs, recs, v0, wav, wavc, refl = mgk.flow_setup(P, r)
        ops.append(pm.local.LSM(z, x, t, srcs, recs, v0, wav, wavc, mode="analytic"))
    return ops, refl


def bcast(pm, a):
    return pm.DistributedArray.to_dist(a, partition=pm.Partition.BROADCAST)


@pytest.mark.gpu
def test_lsqr_tutorial_flow_matches_scipy(pm):
    """tutorials/lsm.py's operator (all sources in one MPIVStack), 100 iterations: scipy's image within TOL_FACTOR
    times the fixture's spread (scipy's loop under a 4-ulp jitter per iteration)"""
    lsms, refl = flow_ops(pm, 1, None)
    Op = pm.MPIVStack([lsms[0].Demop])
    d = Op @ bcast(pm, refl.ravel())
    x, istop, itn, *_ = pm.lsqr(Op, d, x0=bcast(pm, np.zeros(Op.shape[1])), niter=mgl.FLOW_NITER)
    assert istop == int(GOLD["flow/istop"]) and itn == int(GOLD["flow/itn"])
    xg = GOLD["flow/x"]
    tol = TOL_FACTOR * float(GOLD["flow/spread"])
    err = np.abs(host(x.asarray()) - xg).max() / np.abs(xg).max()
    assert err <= tol, (err, tol)


@pytest.mark.gpu
def test_lsm_solve_equals_lsqr_on_vstack(pm):
    """LSM.solve inverts one rank's sources: the same body as lsqr(MPIVStack([Demop])) on a one-rank communicator,
    so the same bits; scipy's image within TOL_FACTOR times the fixture's spread"""
    (lsm,), refl = flow_ops(pm, 2, 0)
    one = pm.Comm(rank=0, size=1)
    Op = pm.MPIVStack([lsm.Demop], base_comm=one)
    d = Op @ pm.DistributedArray.to_dist(refl.ravel(), base_comm=one, partition=pm.Partition.BROADCAST)
    dh = host(d.asarray())
    img = lsm.solve(dh, niter=mgl.FLOW_NITER)
    x0 = pm.DistributedArray.to_dist(np.zeros(Op.shape[1]), base_comm=one, partition=pm.Partition.BROADCAST)
    ref = pm.lsqr(Op, d, x0=x0, niter=mgl.FLOW_NITER)[0]
    assert tuple(img.shape) == tuple(lsm.Demop.dims) and img.is_cuda
    np.testing.assert_array_equal(host(img).ravel(), host(ref.asarray()))
    xg = GOLD["lsm/x"]
    err = np.abs(host(img).ravel() - xg).max() / np.abs(xg).max()
    assert err <= TOL_FACTOR * float(GOLD["lsm/spread"]), err
    # solver=cgls: cgls's own bits
    img_c = lsm.solve(dh, solver=pm.cgls, niter=20)
    ref_c = pm.cgls(Op, d, x0=x0, niter=20)[0]
    np.testing.assert_array_equal(host(img_c).ravel(), host(ref_c.asarray()))
    with pytest.raises(NotImplementedError, match="solver"):
        lsm.solve(dh, solver=lambda *a, **k: None)
    with pytest.raises(ValueError, match="values"):
        lsm.solve(dh[:-1])


@pytest.mark.gpu
def test_lsqr_two_ranks():
    """``on_ranks`` at P = 2: SCATTER and BROADCAST models, fixtures, graph vs step() bits"""
    needs_gpus(2)
    run_on_ranks("test_lsqr", 2)


def on_ranks(pm, comm):
    """LSQR at world size P = 2, one rank per GPU:

    - MPIBlockDiag (SCATTER model), rank r holding diagonal block r of a fixture case (P = 2 = NBLK): istop and the
      iteration count exactly, x, var, the scalars and the cost within the single-GPU tolerances of test_lsqr.py;
    - MPIVStack (BROADCAST model) of both blocks: against the same solve on a one-rank communicator in this process.
      Every rank updates the whole model but adds only its share to |dk|^2: a doubled ddnorm would move acond by a
      factor sqrt(2).  The scalars are allowed 0.1 (of themselves; r1norm, r2norm of cost[0], arnorm of anorm * cost[0]),
      x 1e-4 of its largest entry: the two solves differ in the order of the all-reduced sums only, and the damped
      fixture's spreads under a 4-ulp jitter per iteration are 1.2e-2 for acond and 7.7e-6 for x;
    - both: the graph-replayed run and a step() loop give identical bits at P = 2.
    """
    from pylops_mpi_b200.optimization.cls_basic import LSQR
    rank, P = comm.Get_rank(), comm.Get_size()
    assert P == mgl.NBLK, P

    def block(name, r):
        A = GOLD[f"{name}/A"]
        m, n = A.shape[0] // mgl.NBLK, A.shape[1] // mgl.NBLK
        return np.ascontiguousarray(A[r * m:(r + 1) * m, r * n:(r + 1) * n])

    def step_loop(Op, y, x0, kw):
        s = LSQR(Op)
        x = s.setup(y=y, x0=x0, **kw)
        while s.iiter < kw["niter"] and s.istop == 0:
            x = s.step(x)
        s.finalize()
        return (x, s.istop, s.iiter, s.r1norm, s.r2norm, s.anorm, s.acond, s.arnorm, s.xnorm, s.var, s.cost)

    def flat(out):
        return [host(o.asarray()) if hasattr(o, "asarray") else np.asarray(o) for o in out]

    def same_bits(a, b, what):
        for i, (g, r) in enumerate(zip(flat(a), flat(b))):
            np.testing.assert_array_equal(g, r, err_msg=f"[rank {rank}] {what}: output {i}")

    for name in ("inconsistent", "illcond", "damped", "complex"):
        kw, has_x0 = params(name)
        Op = pm.MPIBlockDiag([pm.MatrixMult(block(name, rank))])
        y = pm.DistributedArray.to_dist(GOLD[f"{name}/b"])
        x0 = pm.DistributedArray.to_dist(GOLD[f"{name}/x0"]) if has_x0 else None
        s = LSQR(Op)
        out = s.solve(y, x0, **kw)
        assert s.graph_error is None and s.graph_replays > 0, s.graph_error
        x, istop, itn, r1, r2, anorm, acond, arnorm, xnorm, var, cost = out
        assert istop == int(GOLD[f"{name}/istop"]) and itn == int(GOLD[f"{name}/itn"]), (rank, name, istop, itn)
        xg, vg = GOLD[f"{name}/x"], GOLD[f"{name}/var"]
        np.testing.assert_allclose(host(x.asarray()), xg, rtol=0, atol=tol(name, 0) * np.abs(xg).max())
        np.testing.assert_allclose(host(var.asarray()), vg, rtol=0, atol=tol(name, 1) * np.abs(vg).max())
        for i, (k, got) in enumerate(zip(SCALARS, (r1, r2, anorm, acond, arnorm, xnorm))):
            assert abs(got - float(GOLD[f"{name}/{k}"])) <= tol(name, 2 + i) * scalar_scale(name, k), (rank, name, k)
        cg = GOLD[f"{name}/cost"]
        np.testing.assert_allclose(cost, cg, rtol=0, atol=tol(name, 8) * cg[0])
        same_bits(step_loop(Op, y, x0, kw), out, f"blockdiag {name} step vs graph")

    one = pm.Comm(rank=0, size=1)
    for name in ("inconsistent", "damped"):
        kw, _ = params(name)
        kw["niter"] = min(kw["niter"], 40)
        blocks = [block(name, r) for r in range(P)]
        b = GOLD[f"{name}/b"]
        Op = pm.MPIVStack([pm.MatrixMult(blocks[rank])])
        y = pm.DistributedArray.to_dist(b)
        s = LSQR(Op)
        out = s.solve(y, None, **kw)
        assert s.graph_error is None and s.graph_replays > 0, s.graph_error
        same_bits(step_loop(Op, y, None, kw), out, f"vstack {name} step vs graph")
        Op1 = pm.MPIVStack([pm.MatrixMult(np.vstack(blocks))], base_comm=one)
        ref = pm.lsqr(Op1, pm.DistributedArray.to_dist(b, base_comm=one), niter=kw["niter"], damp=kw["damp"],
                      atol=kw["atol"], btol=kw["btol"], conlim=kw["conlim"])
        assert out[1] == ref[1] and out[2] == ref[2], (rank, name, out[1:3], ref[1:3])
        np.testing.assert_allclose(host(out[0].asarray()), host(ref[0].asarray()), rtol=0,
                                   atol=1e-4 * np.abs(host(ref[0].asarray())).max(), err_msg=f"[rank {rank}] {name} x")
        c0 = float(ref[10][0])
        for i, k in enumerate(SCALARS):
            scale = {"r1norm": c0, "r2norm": c0, "arnorm": ref[5] * c0}.get(k, abs(ref[3 + i]))
            assert abs(out[3 + i] - ref[3 + i]) <= 0.1 * scale, (rank, name, k, out[3 + i], ref[3 + i])
