"""Rank-local NonStationaryFilters1D / NonStationaryFilters2D (pylops.signalprocessing inside MPIVStack): estimating
a bank of non-stationary filters from a fixed input.

    forward  y[i] = sum_j h_j[hc + i - j] inp[j]     (h_j interpolated from the model bank)  ==  NSC(model) inp
    adjoint  g_c[k] = sum_(j in S_c) W_c[j] inp[j] d[j + k - hc]

CPU: refshim's restatement against the dense definition (the matrix whose columns are NSC(e_c) inp), the operators'
argument errors, and the fixtures of tests/golden/nsfilters_golden.npz (made by make_golden_nsfilters.py: the
reference's MPIVStack over the restatement; inputs exactly representable, so every dtype must match them bit for
bit).  GPU: b2_nsfilters2d_adjoint through the C ABI, and the operators through the public interface."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_nsfilters as mgf  # noqa: E402
from ns_reference import U, assert_within, axis_w, gamma  # noqa: E402
from fixture_codec import decode, rows_of  # noqa: E402
from op_checks import assert_cgls_replay_matches_steps, guarded_twice, host, needs_gpus, run_on_ranks  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "nsfilters_golden.npz"), allow_pickle=False)


def refshim():
    path = os.path.join(HERE, "golden", "refshim")
    sys.path.insert(0, path)
    try:
        from pylops.signalprocessing import nonstatconvolve1d, nonstatconvolve2d, nonstatfilters
    finally:
        sys.path.remove(path)
    return nonstatconvolve1d, nonstatconvolve2d, nonstatfilters


def dense(kind, inp, bshape, ih):
    """the float64 matrix of the filter estimation: column c is NSC(e_c) inp (the restated convolution)"""
    c1, c2, _ = refshim()
    nb = int(np.prod(bshape))
    M = np.zeros((inp.size, nb))
    for c in range(nb):
        e = np.zeros(nb)
        e[c] = 1.0
        if kind == 1:
            M[:, c] = c1.NonStationaryConvolve1D(inp.size, e.reshape(bshape), ih[0]).matvec(inp.astype(np.float64))
        else:
            M[:, c] = c2.NonStationaryConvolve2D(inp.shape, e.reshape(bshape), *ih).matvec(inp.astype(np.float64))
    return M


def adjoint_ref(d, inp, nf, nh, oh, dh, dt):
    """(g, bound): the float64 adjoint by the definition with weights rounded to dt, and sum |terms|"""
    nx, nz = inp.shape
    Wx, Wz = axis_w(nx, oh[0], dh[0], nf[0]), axis_w(nz, oh[1], dh[1], nf[1])
    hcx, hcz = nh[0] // 2, nh[1] // 2
    dp = np.zeros((nx + nh[0] + 1, nz + nh[1] + 1))            # d padded by the reach of the taps
    dp[hcx:hcx + nx, hcz:hcz + nz] = d
    g, b = np.zeros(nf + nh), np.zeros(nf + nh)
    for a in range(nf[0]):
        for bb in range(nf[1]):
            u = np.outer(Wx[a], Wz[bb]).astype(dt).astype(np.float64) * inp
            for kx in range(nh[0]):
                for kz in range(nh[1]):
                    win = dp[kx:kx + nx, kz:kz + nz]
                    g[a, bb, kx, kz] = np.sum(u * win)
                    b[a, bb, kx, kz] = np.sum(np.abs(u * win))
    return g, b


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hsize,nf,dh,oh", [(1, 1, 1, 0), (5, 2, 4, 1), (7, 5, 3, 2), (41, 3, 6, 4)])
def test_restatement_1d_is_the_definition(hsize, nf, dh, oh):
    _, _, F = refshim()
    rng = np.random.default_rng(hsize + nf)
    inp = rng.standard_normal(23)
    ih = oh + dh * np.arange(nf)
    Op = F.NonStationaryFilters1D(inp, hsize, ih)
    M = dense(1, inp, (nf, hsize), (ih,))
    x, v = rng.standard_normal(nf * hsize), rng.standard_normal(23)
    np.testing.assert_allclose(Op.matvec(x), M @ x, rtol=0, atol=1e-12)
    np.testing.assert_allclose(Op.rmatvec(v), M.T @ v, rtol=0, atol=1e-12)


@pytest.mark.parametrize("nh", [(1, 1), (3, 5), (7, 3)])
@pytest.mark.parametrize("nf,dh,oh", [((1, 1), (1, 1), (0, 3)), ((2, 3), (3, 2), (1, 2)), ((3, 2), (4, 5), (2, 0))])
def test_restatement_2d_is_the_definition(nh, nf, dh, oh):
    _, _, F = refshim()
    rng = np.random.default_rng(nh[0] * 10 + nh[1] + nf[0])
    inp = rng.standard_normal((11, 13))
    ih = (oh[0] + dh[0] * np.arange(nf[0]), oh[1] + dh[1] * np.arange(nf[1]))
    Op = F.NonStationaryFilters2D(inp, nh, *ih)
    M = dense(2, inp, nf + nh, ih)
    x, v = rng.standard_normal(M.shape[1]), rng.standard_normal(M.shape[0])
    np.testing.assert_allclose(Op.matvec(x), M @ x, rtol=0, atol=1e-12)
    np.testing.assert_allclose(Op.rmatvec(v), M.T @ v, rtol=0, atol=1e-12)
    g, _ = adjoint_ref(v.reshape(inp.shape), inp, nf, nh, oh, dh, np.float64)   # the kernel's decomposition
    np.testing.assert_allclose(g.ravel(), M.T @ v, rtol=0, atol=1e-12)


def test_operator_argument_errors():
    import pylops_mpi_b200.local as L
    inp2, inp1 = np.ones((20, 10)), np.ones(30)
    good = dict(inp=inp2, hshape=(5, 3), ihx=[2, 6, 10], ihz=[1, 4])
    for bad in (dict(hshape=(4, 3)), dict(hshape=(5, 2)),                           # even filter sizes
                dict(ihx=[2, 6, 11]), dict(ihz=[1, 4, 8]),                          # irregular
                dict(ihx=[-1, 3, 7]), dict(ihx=[10, 15, 20]), dict(ihz=[5, 10]),    # outside [0, dims)
                dict(ihx=[10, 6, 2]), dict(ihz=[4, 1]),                             # decreasing
                dict(inp=inp1), dict(inp=np.ones((2, 20, 10))), dict(hshape=(5, 3, 1))):
        kw = dict(good)
        kw.update(bad)
        with pytest.raises(ValueError):
            L.NonStationaryFilters2D(kw["inp"], kw["hshape"], kw["ihx"], kw["ihz"])
    for bad in (dict(hsize=4), dict(ih=[2, 6, 11]), dict(ih=[-1, 3]), dict(ih=[20, 30]), dict(ih=[6, 2]),
                dict(inp=inp2)):
        kw = dict(inp=inp1, hsize=5, ih=[2, 6, 10])
        kw.update(bad)
        with pytest.raises(ValueError):
            L.NonStationaryFilters1D(kw["inp"], kw["hsize"], kw["ih"])
    with pytest.raises(NotImplementedError):
        L.NonStationaryFilters2D(inp2 + 1j, (5, 3), [2, 6, 10], [1, 4])
    with pytest.raises(NotImplementedError):
        L.NonStationaryFilters1D(inp1 + 1j, 5, [2, 6, 10])


def case_id(c):
    kind, nh, bank, dt = c
    return f"{mgf.key(kind, nh, bank)}/{dt}"


def test_fixture_inventory():
    want = set()
    for kind, nh, bank, dt in mgf.cases():
        for n in ("y", "ya", "yi", "yai")[:4 if dt == "complex128" else 2]:
            assert GOLD[f"{mgf.key(kind, nh, bank)}/{n}"].dtype == np.int32
            want.add(f"{mgf.key(kind, nh, bank)}/{n}")
    want |= {"flow1/refl", "flow1/d", "flow2/mmig", "flow2/m"}
    for f, names in (("flow1", ("x", "iiter", "cost")), ("flow2", ("x", "iiter", "cost", "heldout"))):
        want |= {f"{f}/cond", f"{f}/spread"} | {f"{f}/P{P}/{k}" for P in (1, 2, 3) for k in names}
        assert GOLD[f"{f}/spread"].shape == (2,) and float(GOLD[f"{f}/spread"].max()) < 1e-10    # reproducible
        for P in (1, 2, 3):
            assert int(GOLD[f"{f}/P{P}/iiter"]) == (mgf.FLOW1_NITER if f == "flow1" else mgf.FLOW2_NITER)
    assert set(GOLD.files) == want


def test_weights_and_clamps_of_the_restated_adjoints():
    """one input sample, one data sample on it, filters of one tap: the adjoint is the sample's weight on every
    filter, which must be the definition's (1 on the end filter outside the nodes; pylops' 0.5 + 0.5 clamp in 2-D)"""
    _, _, F = refshim()
    for nf, dh, oh in ((1, 1, 0), (1, 1, 5), (2, 3, 1), (4, 4, 2), (5, 7, 6)):
        ih = oh + dh * np.arange(nf)
        n = max(40, int(ih[-1]) + 1)
        W = axis_w(n, oh, dh, nf)
        for j in range(n):
            e = np.zeros(n)
            e[j] = 1.0
            np.testing.assert_array_equal(F.NonStationaryFilters1D(e, 1, ih).rmatvec(e), W[:, j])
        Wz = axis_w(7, 1, 3, 2)
        for jx in range(0, n, 3):
            for jz in range(7):
                e = np.zeros((n, 7))
                e[jx, jz] = 1.0
                g = F.NonStationaryFilters2D(e, (1, 1), ih, [1, 4]).rmatvec(e.ravel())
                np.testing.assert_allclose(g, np.outer(W[:, jx], Wz[:, jz]).ravel(), rtol=0, atol=1e-15)


def test_flow_inputs_regenerate():
    wav, refl, d = mgf.flow1_inputs()
    np.testing.assert_array_equal(refl, GOLD["flow1/refl"])
    np.testing.assert_array_equal(d, GOLD["flow1/d"])
    assert wav.shape == (len(mgf.FLOW1_IH), 15)
    mmig, m = mgf.flow2_inputs()
    np.testing.assert_array_equal(mmig, GOLD["flow2/mmig"])
    np.testing.assert_array_equal(m, GOLD["flow2/m"])


@pytest.mark.parametrize("case", mgf.cases(), ids=[case_id(c) for c in mgf.cases()])
def test_fixtures_follow_the_restatement_in_every_dtype(case):
    kind, nh, bank, dt = case
    _, _, F = refshim()
    inp, ih, bshape, x, v = mgf.case_inputs(kind, nh, bank, dt)
    plane = int(np.prod(inp.shape[1:]))
    ops = [F.NonStationaryFilters1D(i, nh, ih[0], dtype=dt) if kind == 1 else
           F.NonStationaryFilters2D(i, nh, *ih, dtype=dt) for i in inp]
    y = np.concatenate([op.matvec(x) for op in ops])
    ya = sum(op.rmatvec(v[k * plane:(k + 1) * plane]) for k, op in enumerate(ops))
    gy, gya = decode(GOLD, mgf.key(kind, nh, bank), dt, mgf.ENC)
    np.testing.assert_array_equal(y, gy)
    np.testing.assert_array_equal(ya, gya)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernel through the C ABI
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


def geom(shape, nf, nh, oh, dh):
    return (shape[0], shape[1], nf[0], nf[1], nh[0], nh[1], oh[0], dh[0], oh[1], dh[1])


def work_bytes(pm, g, code):
    import ctypes
    n = ctypes.c_size_t(0)
    assert pm._lib.lib.b2_nsfilters2d_work_bytes(*g, code, ctypes.byref(n)) == 0
    return n.value


def run_adjoint(pm, d_np, inp_np, nf, nh, oh, dh, dt, guard=5):
    """g through the C ABI into a guarded view; returns (g, guards intact, second apply bit-equal, work bytes)"""
    import torch
    code = pm._lib.F32 if dt == np.float32 else pm._lib.F64
    d = torch.as_tensor(np.ascontiguousarray(d_np, dtype=dt)).cuda()
    inp = torch.as_tensor(np.ascontiguousarray(inp_np, dtype=dt)).cuda()
    gm = geom(d_np.shape, nf, nh, oh, dh)
    nw = work_bytes(pm, gm, code)
    work = torch.empty(max(nw, 1), dtype=torch.uint8, device="cuda")
    L = pm._lib
    g, guards_ok, same = guarded_twice(
        lambda gp: L.lib.b2_nsfilters2d_adjoint(L.ctx(), d.data_ptr(), inp.data_ptr(), gp, *gm, work.data_ptr(), nw,
                                                code, L.stream()), int(np.prod(nf + nh)), dt, guard)
    return g.reshape(nf + nh), guards_ok, same, nw


def check_adjoint(pm, shape, nf, nh, oh, dh, dt, seed=0, want_split=None):
    rng = np.random.default_rng(seed)
    d, inp = rng.standard_normal(shape), rng.standard_normal(shape)
    g, guards_ok, repeat_ok, nw = run_adjoint(pm, d, inp, nf, nh, oh, dh, dt)
    assert guards_ok and repeat_ok
    if want_split is not None:
        assert (nw > 0) == want_split
    ref, bnd = adjoint_ref(d.astype(dt).astype(np.float64), inp.astype(dt).astype(np.float64), nf, nh, oh, dh, dt)
    # per filter c, K_c = |S_c| terms: a tap's longest chain is one fma per support point (the part fold adds no more
    # operations than there are points), plus the rounded weight and the rounded product W_c inp of each term
    Wx, Wz = axis_w(shape[0], oh[0], dh[0], nf[0]), axis_w(shape[1], oh[1], dh[1], nf[1])
    K = np.count_nonzero(Wx, 1)[:, None] * np.count_nonzero(Wz, 1)[None, :] + 3
    assert_within(g, ref, gamma(K, dt)[:, :, None, None] * bnd)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("case", [
    ((1, 1), (1, 1), (1, 1), (0, 0), (1, 1)),            # a single point
    ((1, 37), (1, 3), (1, 5), (0, 4), (1, 12)),          # singleton x axis (the 1-D path)
    ((29, 1), (3, 1), (7, 1), (2, 0), (10, 1)),          # singleton z axis
    ((20, 24), (2, 3), (3, 5), (1, 1), (1, 4)),          # small, both ends extrapolated
    ((20, 24), (4, 5), (41, 41), (1, 1), (4, 4)),        # filters larger than the image
    ((70, 130), (3, 4), (33, 65), (5, 7), (30, 40)),     # partial tap tiles and support chunks
], ids=["point", "x1", "z1", "small", "big-filters", "partial-tiles"])
def test_kernel_vs_definition(pm, dt, case):
    shape, nf, nh, oh, dh = case
    check_adjoint(pm, shape, nf, nh, oh, dh, dt, seed=sum(shape))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
def test_kernel_split_and_many_filter_paths(pm, dt):
    # few filters with huge supports: the supports are split into parts and folded
    check_adjoint(pm, (300, 520), (1, 2), (3, 5), (0, 100), (1, 300), dt, seed=1, want_split=True)
    check_adjoint(pm, (260, 300), (2, 3), (7, 9), (60, 20), (140, 130), dt, seed=2, want_split=True)
    # many filters: one part, written straight into the bank
    check_adjoint(pm, (128, 256), (32, 32), (3, 3), (2, 4), (4, 8), dt, seed=3, want_split=False)


@pytest.mark.gpu
def test_kernel_error_codes_leave_output_untouched(pm):
    import torch
    L = pm._lib
    d = torch.randn(20 * 24, dtype=torch.float64, device="cuda")
    inp = torch.randn(20 * 24, dtype=torch.float64, device="cuda")
    nb = 2 * 1 * 3 * 5
    g = torch.full((nb,), 7.25, dtype=torch.float64, device="cuda")
    gm = (20, 24, 2, 1, 3, 5, 1, 10, 0, 1)
    ok = lambda **k: L.lib.b2_nsfilters2d_adjoint(  # noqa: E731
        k.get("ctx", L.ctx()), k.get("d", d.data_ptr()), k.get("inp", inp.data_ptr()), k.get("g", g.data_ptr()),
        *k.get("gm", gm), k.get("work", None), k.get("nw", 0), k.get("code", L.F64), L.stream())
    bad = [dict(ctx=None), dict(d=None), dict(inp=None), dict(g=None), dict(g=d.data_ptr()),
           dict(g=inp.data_ptr() + 8), dict(gm=(0, 24, 2, 1, 3, 5, 1, 10, 0, 1)), dict(gm=(20, 0, 2, 1, 3, 5, 1, 10, 0, 1)),
           dict(gm=(20, 24, 0, 1, 3, 5, 1, 10, 0, 1)), dict(gm=(20, 24, 2, 1, 0, 5, 1, 10, 0, 1)),
           dict(gm=(20, 24, 2, 1, 3, 5, 1, 0, 0, 1)), dict(gm=(20, 24, 2, 1, 3, 5, 1, 10, 0, -1))]
    for k in bad:
        assert ok(**k) == 2002, k                       # B2_ERR_ARG
    assert ok(code=L.C128) == 2001                      # B2_ERR_DTYPE
    # a shape that needs a workspace: none, a short one, and one overlapping the output
    big = (300, 520, 1, 2, 3, 5, 0, 1, 100, 300)
    nw = work_bytes(pm, big, L.F64)
    assert nw > 0
    d2 = torch.randn(300 * 520, dtype=torch.float64, device="cuda")
    w = torch.empty(nw + 64, dtype=torch.uint8, device="cuda")
    for k in (dict(work=None, nw=nw), dict(work=w.data_ptr(), nw=nw - 8), dict(work=g.data_ptr(), nw=nw),
              dict(work=d2.data_ptr(), nw=nw)):
        assert ok(d=d2.data_ptr(), inp=d2.data_ptr(), gm=big, **k) == 2002, k
    torch.cuda.synchronize()
    assert bool((g == 7.25).all())
    assert ok(d=d2.data_ptr(), inp=d2.data_ptr(), gm=big, work=w.data_ptr(), nw=nw) == 0   # d may be inp


# ---------------------------------------------------------------------------------------------------------------
# GPU: the operators
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["float32", "float64"])
def test_forward_equals_the_convolution_bit_for_bit(pm, dt):
    import torch
    rng = np.random.default_rng(5)
    inp2 = rng.standard_normal((37, 53))
    hs2 = rng.standard_normal((3, 4, 9, 7))
    F2 = pm.local.NonStationaryFilters2D(inp2, (9, 7), [2, 14, 26], [3, 15, 27, 39], dtype=dt)
    C2 = pm.local.NonStationaryConvolve2D((37, 53), hs2, [2, 14, 26], [3, 15, 27, 39], dtype=dt)
    tdt = getattr(torch, dt)
    big = torch.as_tensor(rng.standard_normal(hs2.size + 1)).to(tdt).cuda()
    model = big[1:]                                     # a slice: one element off the allocation's alignment
    model.copy_(torch.as_tensor(hs2.ravel()).to(tdt))
    want = C2.matvec(torch.as_tensor(inp2.ravel()).to(tdt).cuda())
    assert torch.equal(F2.matvec(model), want)
    inp1, hs1 = rng.standard_normal(101), rng.standard_normal((4, 11))
    F1 = pm.local.NonStationaryFilters1D(inp1, 11, [5, 30, 55, 80], dtype=dt)
    C1 = pm.local.NonStationaryConvolve1D(101, hs1, [5, 30, 55, 80], dtype=dt)
    big = torch.as_tensor(rng.standard_normal(hs1.size + 1)).to(tdt).cuda()
    big[1:] = torch.as_tensor(hs1.ravel()).to(tdt)
    assert torch.equal(F1.matvec(big[1:]), C1.matvec(torch.as_tensor(inp1).to(tdt).cuda()))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
def test_1d_adjoint_vs_dense_matrix(pm, dt):
    import torch
    rng = np.random.default_rng(9)
    inp, v = rng.standard_normal(301), rng.standard_normal(301)
    ih = 7 + 40 * np.arange(6)
    Op = pm.local.NonStationaryFilters1D(inp, 41, ih, dtype=dt.__name__)
    M = dense(1, inp.astype(dt), (6, 41), (ih,))
    got = host(Op.rmatvec(torch.as_tensor(v.astype(dt)).cuda())).astype(np.float64)
    ref, bnd = M.T @ v.astype(dt), np.abs(M.T) @ np.abs(v.astype(dt))
    assert np.all(np.abs(got - ref) <= 2 * 310 * U[dt] * bnd)


def vstack_ops(pm, kind, nh, bank, dt):
    """the operators of the generator's MPIVStack, of the same dtype (complex128 included)"""
    inp, ih, _, _, _ = mgf.case_inputs(kind, nh, bank, dt)
    if kind == 1:
        return [pm.local.NonStationaryFilters1D(i, nh, ih[0], dtype=dt) for i in inp]
    return [pm.local.NonStationaryFilters2D(i, nh, *ih, dtype=dt) for i in inp]


@pytest.mark.gpu
@pytest.mark.parametrize("case", mgf.cases(), ids=[case_id(c) for c in mgf.cases()])
def test_operator_vs_reference_fixtures(pm, case):
    kind, nh, bank, dt = case
    _, _, _, x, v = mgf.case_inputs(kind, nh, bank, dt)
    Op = pm.MPIVStack(vstack_ops(pm, kind, nh, bank, dt), dtype=dt)
    got = host((Op @ pm.DistributedArray.to_dist(x, partition=pm.Partition.BROADCAST)).asarray())
    gota = host((Op.H @ pm.DistributedArray.to_dist(v)).asarray())
    assert got.dtype == np.dtype(dt) and gota.dtype == np.dtype(dt)
    gy, gya = decode(GOLD, mgf.key(kind, nh, bank), dt, mgf.ENC)
    np.testing.assert_array_equal(got, gy)
    np.testing.assert_array_equal(gota, gya)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["float64", "float32", "complex128"])
def test_operator_dottest(pm, dt):
    from pylops_mpi_b200.utils.dottest import dottest
    rng = np.random.default_rng(8)
    rdt = "float32" if dt == "float32" else "float64"
    ops = [pm.local.NonStationaryFilters2D(rng.standard_normal((31, 47)), (7, 11), [2, 12, 22], [3, 13, 23, 33],
                                           dtype=rdt) for _ in range(3)]
    Op = pm.MPIVStack(ops, dtype=dt)
    m, n = Op.shape
    cx = dt == "complex128"
    u = rng.standard_normal(n) + (1j * rng.standard_normal(n) if cx else 0)
    v = rng.standard_normal(m) + (1j * rng.standard_normal(m) if cx else 0)
    assert dottest(Op, pm.DistributedArray.to_dist(u.astype(dt), partition=pm.Partition.BROADCAST),
                   pm.DistributedArray.to_dist(v.astype(dt)), rtol=1e-4 if dt == "float32" else 1e-12)


@pytest.mark.gpu
def test_operator_attributes_dtypes_and_out(pm):
    import torch
    rng = np.random.default_rng(4)
    inp = rng.standard_normal((20, 9))
    Op = pm.local.NonStationaryFilters2D(inp, (5, 7), [2, 6, 10], [1, 4], dtype="float32", engine="cuda",
                                         num_threads_per_blocks=(8, 8))
    assert Op.dims == (3, 2, 5, 7) and Op.dimsd == (20, 9) and Op.shape == (180, 210) and Op.dtype == np.float32
    assert (Op.nfilt, Op.nh, Op.hc, Op.oh, Op.dh) == ((3, 2), (5, 7), (2, 3), (2, 1), (4, 3))
    O1 = pm.local.NonStationaryFilters1D(inp[:, 0], 5, [3])
    assert O1.dims == (1, 5) and O1.dimsd == (20,) and O1.shape == (20, 5) and O1.dh == 1
    op64 = pm.local.NonStationaryFilters2D(inp, (5, 7), [2, 6, 10], [1, 4])
    # a complex operator computes in its real dtype and returns complex results
    opc = pm.local.NonStationaryFilters2D(inp, (5, 7), [2, 6, 10], [1, 4], dtype="complex128")
    assert opc.dtype == np.complex128
    for f, fc, nin in ((op64.matvec, opc.matvec, 210), (op64.rmatvec, opc.rmatvec, 180)):
        xr = torch.as_tensor(rng.standard_normal(nin)).cuda()
        yc = fc(xr)
        assert yc.dtype == torch.complex128 and torch.equal(yc.real, f(xr)) and bool((yc.imag == 0).all())
        xc = xr + 1j * torch.as_tensor(rng.standard_normal(nin)).cuda()
        assert torch.equal(fc(xc), f(xc))
    # a float32 operator uses inp rounded to float32
    M = dense(2, inp.astype(np.float32), (3, 2, 5, 7), ([2, 6, 10], [1, 4]))
    x = rng.standard_normal(210).astype(np.float32)
    np.testing.assert_allclose(host(Op.matvec(torch.as_tensor(x).cuda())), M @ x, rtol=0,
                               atol=1e-5 * np.abs(M).sum(1).max())


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["float32", "float64"])
def test_cgls_graph_replay_matches_step_loop(pm, dt):
    rng = np.random.default_rng(12)
    ops = [pm.local.NonStationaryFilters2D(rng.standard_normal((300, 520)), (5, 5), [0], [100, 400], dtype=dt)
           for _ in range(2)]
    assert all(op._work is not None for op in ops)          # the split path, with its workspace, is captured
    Op = pm.MPIVStack(ops)
    y = Op @ pm.DistributedArray.to_dist(rng.standard_normal(Op.shape[1]).astype(dt),
                                         partition=pm.Partition.BROADCAST)
    x0 = pm.DistributedArray.to_dist(np.zeros(Op.shape[1], dtype=dt), partition=pm.Partition.BROADCAST)
    assert_cgls_replay_matches_steps(pm, Op, y, x0, 15, 10)


def flow_tolerance(f):
    """(x, cost) relative tolerances of flow f: the cgls run summed in another order than pylops' moves by about what
    a 4-ulp jitter of every apply moves the reference's own run (``spread``), and by no less than cond * 2^-53
    (``cond``, the stacked operator's condition number); the test allows 100 and 10 times those"""
    floor = 10 * float(GOLD[f"{f}/cond"]) * 2.0 ** -53
    return tuple(max(100 * float(s), floor) for s in GOLD[f"{f}/spread"])


def flow_ops(pm, kind, P):
    """the operators of P ranks' MPIVStacks, in rank order, as one rank's"""
    if kind == 1:
        inps = GOLD["flow1/refl"]
        return [pm.local.NonStationaryFilters1D(i, 15, mgf.FLOW1_IH) for i in inps]
    inps = GOLD["flow2/mmig"][:mgf.FLOW2_NTRAIN]
    return [pm.local.NonStationaryFilters2D(i, mgf.FLOW2_NH, mgf.mg2.FLOW_IHX, mgf.mg2.FLOW_IHZ) for i in inps]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [1, 2], ids=["wavelet-1d", "deblur-2d"])
@pytest.mark.parametrize("P", [1, 2, 3])
def test_estimation_flows_vs_reference(pm, kind, P):
    """cgls on MPIVStack([NonStationaryFilters]) from x0 = 0; the 2-D flow's filter applied to the held-out image"""
    f = f"flow{kind}"
    Op = pm.MPIVStack(flow_ops(pm, kind, P))
    d = GOLD["flow1/d"] if kind == 1 else GOLD["flow2/m"][:mgf.FLOW2_NTRAIN].ravel()
    x0 = pm.DistributedArray.to_dist(np.zeros(Op.shape[1]), partition=pm.Partition.BROADCAST)
    niter = mgf.FLOW1_NITER if kind == 1 else mgf.FLOW2_NITER
    x, _, iiter, _, _, cost = pm.cgls(Op, pm.DistributedArray.to_dist(d), x0=x0, niter=niter, tol=0.0)
    assert iiter == int(GOLD[f"{f}/P{P}/iiter"])
    xtol, ctol = flow_tolerance(f)
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"{f}/P{P}/cost"], rtol=ctol)
    gx = GOLD[f"{f}/P{P}/x"]
    xh = host(x.asarray())
    np.testing.assert_allclose(xh, gx, rtol=0, atol=xtol * np.abs(gx).max())
    if kind == 2:
        import torch
        bshape = (len(mgf.mg2.FLOW_IHX), len(mgf.mg2.FLOW_IHZ)) + mgf.FLOW2_NH
        C = pm.local.NonStationaryConvolve2D((mgf.mg2.FLOW_NX, mgf.mg2.FLOW_NZ), xh.reshape(bshape),
                                             mgf.mg2.FLOW_IHX, mgf.mg2.FLOW_IHZ)
        held = host(C.matvec(torch.as_tensor(GOLD["flow2/mmig"][-1].ravel()).cuda()))
        gh = GOLD[f"flow2/P{P}/heldout"]
        np.testing.assert_allclose(held, gh, rtol=0, atol=2 * xtol * np.abs(gh).max())


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [1, 2])
def test_multi_rank_fixtures(nproc):
    needs_gpus(nproc)
    run_on_ranks("test_nsfilters", nproc)


def on_ranks(pm, comm):
    """each rank's MPIVStack of NonStationaryFilters1D / 2D against its slice of the gathered fixtures, and the
    two estimation flows against their fixtures"""
    rank, P = comm.Get_rank(), comm.Get_size()
    rows = rows_of(P, mgf.NI)
    k0 = sum(rows[:rank])

    for kind, nh, bank, dt in mgf.cases():
        inp, ih, _, x, v = mgf.case_inputs(kind, nh, bank, dt)
        plane = int(np.prod(inp.shape[1:]))
        mine = inp[k0:k0 + rows[rank]]
        ops = ([pm.local.NonStationaryFilters1D(i, nh, ih[0], dtype=dt) for i in mine] if kind == 1 else
               [pm.local.NonStationaryFilters2D(i, nh, *ih, dtype=dt) for i in mine])
        Op = pm.MPIVStack(ops, dtype=dt)
        ls = [(r * plane,) for r in rows]
        gy, gya = decode(GOLD, mgf.key(kind, nh, bank), dt, mgf.ENC)
        name = f"{mgf.key(kind, nh, bank)}/{dt}"
        y = (Op @ pm.DistributedArray.to_dist(x, partition=pm.Partition.BROADCAST)).local_array.cpu().numpy()
        np.testing.assert_array_equal(y, gy[k0 * plane:(k0 + rows[rank]) * plane], err_msg=f"[rank {rank}] {name}/y")
        ya = (Op.H @ pm.DistributedArray.to_dist(v, local_shapes=ls)).local_array.cpu().numpy()
        np.testing.assert_array_equal(ya, gya, err_msg=f"[rank {rank}] {name}/ya")

    # the estimation flows: cgls over this rank's inputs, the bank all-reduced
    for kind in (1, 2):
        f = f"flow{kind}"
        if kind == 1:
            inps, d, niter = GOLD["flow1/refl"], GOLD["flow1/d"], mgf.FLOW1_NITER
        else:
            inps, niter = GOLD["flow2/mmig"][:mgf.FLOW2_NTRAIN], mgf.FLOW2_NITER
            d = GOLD["flow2/m"][:mgf.FLOW2_NTRAIN].ravel()
        fr = rows_of(P, len(inps))
        f0 = sum(fr[:rank])
        plane = int(np.prod(inps.shape[1:]))
        ops = [pm.local.NonStationaryFilters1D(i, 15, mgf.FLOW1_IH) if kind == 1 else
               pm.local.NonStationaryFilters2D(i, mgf.FLOW2_NH, mgf.mg2.FLOW_IHX, mgf.mg2.FLOW_IHZ)
               for i in inps[f0:f0 + fr[rank]]]
        Op = pm.MPIVStack(ops)
        x0 = pm.DistributedArray.to_dist(np.zeros(Op.shape[1]), partition=pm.Partition.BROADCAST)
        dd = pm.DistributedArray.to_dist(d, local_shapes=[(r * plane,) for r in fr])
        x, _, iiter, _, _, cost = pm.cgls(Op, dd, x0=x0, niter=niter, tol=0.0)
        assert iiter == int(GOLD[f"{f}/P{P}/iiter"])
        xtol, ctol = flow_tolerance(f)
        np.testing.assert_allclose(np.asarray(cost), GOLD[f"{f}/P{P}/cost"], rtol=ctol, err_msg=f"[rank {rank}] {f} cost")
        gx = GOLD[f"{f}/P{P}/x"]
        np.testing.assert_allclose(x.local_array.cpu().numpy(), gx, rtol=0, atol=xtol * np.abs(gx).max(),
                                   err_msg=f"[rank {rank}] {f} x")
