"""Rank-local NonStationaryConvolve3D (pylops.signalprocessing inside MPIBlockDiag) and 3-D image-domain least-squares
migration with point-spread functions.

    h_j = sum_(a,b,e) T(wz_e(jz) wy_b(jy) wx_a(jx)) hs[a, b, e]     trilinear in the bank (end filters outside nodes)
    forward y[i] = sum_j h_j[hc + i - j] x[j],  adjoint the transpose

CPU: refshim's restatement against that definition, the interpolation weights, the operator's argument errors, and
the fixtures of tests/golden/nsconvolve3d_golden.npz (made by make_golden_nsconvolve3d.py: the reference's
MPIBlockDiag and cgls over the restatement; operator inputs exactly representable, so every dtype must match them
bit for bit).  GPU: b2_nsconvolve3d through the C ABI, and the operator through the public interface."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_nsconvolve3d as mg3  # noqa: E402
from ns_reference import axis_weights, c_ns, check_close, ns_matrix, point_weights, reference, run_kernel  # noqa: E402
from fixture_codec import decode, rows_of  # noqa: E402
from op_checks import assert_cgls_replay_matches_steps, assert_rejected, host, needs_gpus, run_on_ranks  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "nsconvolve3d_golden.npz"), allow_pickle=False)


def refshim():
    return mg3.refshim_modules()[2]


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nh", [(1, 1, 1), (3, 5, 1), (5, 1, 3)])
@pytest.mark.parametrize("nf,dh,oh", [((1, 1, 1), (1, 1, 1), (0, 3, 2)), ((2, 3, 2), (3, 2, 4), (1, 2, 0)),
                                      ((3, 2, 2), (2, 5, 1), (0, 0, 3))])
def test_refshim_restatement_is_the_definition(nh, nf, dh, oh):
    NS3 = refshim()
    rng = np.random.default_rng(nh[0] * 100 + nh[1] * 10 + nh[2] + nf[0])
    hs = rng.standard_normal(nf + nh)
    ih = [o + d * np.arange(f) for o, d, f in zip(oh, dh, nf)]
    dims = (6, 11, 7)
    Op = NS3(dims, hs, *ih)
    M = ns_matrix(hs, dims, oh, dh)
    x = rng.standard_normal(int(np.prod(dims)))
    np.testing.assert_allclose(Op.matvec(x), M @ x, rtol=0, atol=1e-12)
    np.testing.assert_allclose(Op.rmatvec(x), M.T @ x, rtol=0, atol=1e-12)


@pytest.mark.parametrize("nf,dh,oh", [(1, 1, 0), (1, 1, 5), (2, 3, 1), (4, 4, 2), (5, 7, 6)])
def test_interpolation_weights_and_clamps(nf, dh, oh):
    NS3 = refshim()
    for j in range(40):
        l, r, wl, wr = NS3.weights(j, oh, dh, nf)
        want = axis_weights(j, oh, dh, nf)
        if j <= oh or j >= oh + dh * (nf - 1):                     # at or outside the end nodes
            end = 0 if j <= oh else nf - 1
            assert sorted(want) == [end] and want[end] == 1.0
            if j < oh or j > oh + dh * (nf - 1):                  # pylops' clamp: 0.5 and 0.5 on the end filter
                assert (l, r, wl, wr) == (end, end, 0.5, 0.5)
        else:
            assert l == int(np.floor((j - oh) / dh)) and r == l + 1 and wl + wr == 1.0
            assert wr == (j - oh) / dh - l and wl == 1.0 - wr
            assert {k: w for k, w in ((l, wl), (r, wr)) if w != 0.0} == want
    # the interpolated filter: pylops' eight-term sum equals the definition within float64 rounding
    rng = np.random.default_rng(nf)
    hs = rng.standard_normal((nf, 2, 3, 3, 1, 3))
    Op = NS3((40, 9, 12), hs, oh + dh * np.arange(nf), [2, 6], [1, 5, 9])
    for jx in range(0, 40, 3):
        for jy in range(0, 9, 2):
            for jz in range(12):
                want = sum(W * hs[c] for c, W in point_weights((jx, jy, jz), (oh, 2, 1), (dh, 4, 4), (nf, 2, 3),
                                                                np.float64))
                np.testing.assert_allclose(Op.interpolate_h(jx, jy, jz), want, rtol=0, atol=1e-15)


def test_operator_argument_errors():
    import pylops_mpi_b200.local as L
    NSC = L.NonStationaryConvolve3D
    hs = np.ones((3, 2, 2, 5, 3, 1))
    good = dict(dims=(20, 10, 8), hs=hs, ihx=[2, 6, 10], ihy=[1, 4], ihz=[0, 7])
    for bad in (dict(hs=np.ones((3, 2, 2, 4, 3, 1))), dict(hs=np.ones((3, 2, 2, 5, 2, 1))),   # even filter sizes
                dict(hs=np.ones((3, 2, 2, 5, 3, 2))),
                dict(ihx=[2, 6, 11]), dict(ihy=[1, 4, 8]), dict(ihz=[0, 3, 7]),                # irregular, count
                dict(ihx=[2, 6]), dict(ihy=[1]), dict(ihz=[0, 3, 6]),                          # count mismatch
                dict(ihx=[-1, 3, 7]), dict(ihx=[10, 15, 20]), dict(ihy=[5, 10]), dict(ihz=[1, 8]),  # outside dims
                dict(ihx=[10, 6, 2]), dict(ihy=[4, 1]), dict(ihz=[7, 0]),                      # decreasing
                dict(hs=np.ones((3, 2, 5, 3, 1))), dict(hs=np.ones((1, 3, 2, 2, 5, 3, 1))),     # not 6-D
                dict(dims=(20, 10)), dict(dims=(20, 10, 8, 1)), dict(dims=(200,))):
        kw = dict(good)
        kw.update(bad)
        with pytest.raises(ValueError):
            NSC(kw["dims"], kw["hs"], kw["ihx"], kw["ihy"], kw["ihz"])
    with pytest.raises(NotImplementedError):
        NSC((20, 10, 8), hs + 1j, [2, 6, 10], [1, 4], [0, 7])


def test_fixture_inventory():
    want = set()
    for nh, bank, dt in mg3.cases():
        k = mg3.key(nh, bank)
        for n in ("y", "ya", "yi", "yai")[:4 if dt == "complex128" else 2]:
            assert GOLD[f"{k}/{n}"].dtype == np.int32 and GOLD[f"{k}/{n}"].shape == (mg3.NV * mg3.NX * mg3.NY * mg3.NZ,)
            want.add(f"{k}/{n}")
    ncomplex = sum(dt == "complex128" for _, _, dt in mg3.cases())
    assert ncomplex >= 1 and len(want) == 2 * len(mg3.NHS) * len(mg3.BANKS) + 2 * ncomplex
    flows = {f"flow/P{P}/{k}" for P in (1, 2, 3) for k in ("x", "iiter", "cost")}
    assert sorted(GOLD.files) == sorted(want | flows | {"flow/hs", "flow/mmig", "flow/cond", "flow/spread"})
    dims = (mg3.NX, mg3.NY, mg3.NZ)
    assert sum(max(nh[d] > dims[d] for nh in mg3.NHS) for d in range(3)) >= 2        # larger than the volume
    assert any(len(set(nh)) > 1 for nh in mg3.NHS) and min(min(nh) for nh in mg3.NHS) == 1
    assert max(min(b[0]) for b in mg3.BANKS) >= 3                                      # interior points: 8 filters
    for P in (1, 2, 3):
        assert int(GOLD[f"flow/P{P}/iiter"]) == mg3.FLOW_NITER
    assert GOLD["flow/spread"].shape == (2,) and float(GOLD["flow/spread"].max()) < 1e-9          # reproducible
    assert GOLD["flow/hs"].shape == (len(mg3.FLOW_IHY), len(mg3.FLOW_IHX), len(mg3.FLOW_IHZ)) + mg3.FLOW_NH


def case_id(c):
    nh, (nf, dh), dt = c
    return "nh{}x{}x{}/nf{}x{}x{}/dh{}x{}x{}/".format(*nh, *nf, *dh) + dt


def volumes(a):
    n = mg3.NX * mg3.NY * mg3.NZ
    return [a[k * n:(k + 1) * n] for k in range(mg3.NV)]


@pytest.mark.parametrize("case", mg3.cases(), ids=[case_id(c) for c in mg3.cases()])
def test_fixtures_follow_the_restatement_in_every_dtype(case):
    NS3 = refshim()
    nh, bank, dt = case
    hs, ih, x, v = mg3.case_inputs(nh, bank, dt)
    ops = [NS3((mg3.NX, mg3.NY, mg3.NZ), hs[k], *ih, dtype=dt) for k in range(mg3.NV)]
    y = np.concatenate([op.matvec(s) for op, s in zip(ops, volumes(x))])
    ya = np.concatenate([op.rmatvec(s) for op, s in zip(ops, volumes(v))])
    gy, gya = decode(GOLD, mg3.key(nh, bank), dt, mg3.ENC)
    assert y.dtype == np.dtype(dt) and gy.dtype == np.dtype(dt)
    np.testing.assert_array_equal(y, gy)
    np.testing.assert_array_equal(ya, gya)


def test_flow_psfs_follow_the_restated_kirchhoff():
    kirchhoff3d, _, _ = mg3.refshim_modules()
    z, x, t, srcs, recs, vel, wav, wavc, y = mg3.flow_geometry()
    K = kirchhoff3d.Kirchhoff(z, x, t, srcs, recs, vel, wav, wavc, y=y, mode="analytic")
    m_psf, m_true = mg3.flow_models()
    img = K.rmatvec(K.matvec(m_psf.ravel())).reshape(mg3.FLOW_NY, mg3.FLOW_NX, mg3.FLOW_NZ)
    np.testing.assert_array_equal(mg3.psf_windows(img), GOLD["flow/hs"])
    n = mg3.FLOW_NY * mg3.FLOW_NX * mg3.FLOW_NZ
    np.testing.assert_array_equal(K.rmatvec(K.matvec(m_true[1].ravel())), GOLD["flow/mmig"][n:2 * n])


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernel through the C ABI
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


# singleton axes, tiles that are not full along every axis (x tiles of 4 / 2 / 1 planes, y of 32, z of 64)
SHAPES = [(1, 1, 1), (1, 1, 37), (1, 29, 1), (7, 1, 1), (3, 5, 7), (5, 33, 3), (2, 7, 70), (6, 35, 5)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("nh", [(1, 1, 1), (3, 5, 3), (5, 3, 7), (9, 7, 5)], ids=lambda v: "nh{}x{}x{}".format(*v))
def test_kernel_vs_matrix(pm, dt, nh):
    rng = np.random.default_rng(nh[0] * 100 + nh[1] * 10 + nh[2])
    for dims in SHAPES:
        for nf, dh, oh in (((1, 1, 1), (1, 1, 1), (0, 0, 0)), ((2, 3, 2), (3, 4, 2), (0, 1, 1)),
                           ((3, 2, 2), (2, 7, 3), (1, 2, 0)), ((2, 2, 2), (1, 1, 1), (0, 0, 0))):
            oh = tuple(min(o, d - 1) for o, d in zip(oh, dims))
            nf = tuple(min(f, 1 + (d - 1 - o) // s) for f, d, o, s in zip(nf, dims, oh, dh))
            hs = rng.standard_normal(nf + nh).astype(dt)
            for ni in (1, 2):
                x = rng.standard_normal(dims + (ni,)).astype(dt)
                for adjoint in (False, True):
                    y, guards, same = run_kernel(pm, x, hs, oh, dh, adjoint, dt)
                    assert guards and same, (dims, nf, adjoint, ni)
                    check_close(y, x, hs, oh, dh, adjoint, dt)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("case", ["65x3x65/steps", "3x129x9/steps", "17x33x17/small", "31x1x31/chunks"])
def test_kernel_large_filters_in_chunks(pm, dt, case):
    """filters larger than one chunk of taps and larger than the volume, steps that do not divide dims"""
    nh, dims, nf, dh = {"65x3x65/steps": ((65, 3, 65), (18, 5, 24), (2, 1, 3), (11, 1, 9)),
                        "3x129x9/steps": ((3, 129, 9), (6, 40, 10), (2, 3, 2), (3, 17, 7)),
                        "17x33x17/small": ((17, 33, 17), (12, 12, 12), (1, 1, 1), (1, 1, 1)),
                        "31x1x31/chunks": ((31, 1, 31), (20, 3, 36), (3, 2, 4), (7, 1, 9))}[case]
    rng = np.random.default_rng(len(case) + nh[1])
    hs = rng.standard_normal(nf + nh).astype(dt)
    x = rng.standard_normal(dims + (1,)).astype(dt)
    for adjoint in (False, True):
        y, guards, same = run_kernel(pm, x, hs, (1, 0, 2), dh, adjoint, dt)
        assert guards and same
        check_close(y, x, hs, (1, 0, 2), dh, adjoint, dt)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_kernel_singleton_axis_is_the_2d_kernel(pm, dt, axis):
    """a volume with one sample and one filter (of one tap) along ``axis`` is NonStationaryConvolve2D on the other
    two axes: both kernels within the rounding bound of the same float64 product"""
    rng = np.random.default_rng(31 + axis)
    dims2, nf2, nh2, oh2, dh2 = (37, 70), (3, 4), (7, 9), (2, 3), (13, 19)
    hs2 = rng.standard_normal(nf2 + nh2).astype(dt)
    x2 = rng.standard_normal(dims2 + (2,)).astype(dt)
    ins = lambda t, v: t[:axis] + (v,) + t[axis:]         # noqa: E731
    hs3 = np.expand_dims(np.expand_dims(hs2, axis), 3 + axis)
    x3 = x2.reshape(ins(dims2, 1) + (2,))
    oh3, dh3 = ins(oh2, 0), ins(dh2, 1)
    L = pm._lib
    import torch
    for adjoint in (False, True):
        y3, guards, same = run_kernel(pm, x3, hs3, oh3, dh3, adjoint, dt)
        assert guards and same
        xd = torch.as_tensor(x2.ravel()).cuda()
        yd = torch.empty_like(xd)
        hd = torch.as_tensor(hs2).cuda()
        assert L.lib.b2_nsconvolve2d(L.ctx(), xd.data_ptr(), yd.data_ptr(), *dims2, 2, hd.data_ptr(), *nf2, *nh2,
                                     oh2[0], dh2[0], oh2[1], dh2[1], int(adjoint), L.F32 if dt == np.float32 else L.F64,
                                     L.stream()) == 0
        y2 = host(yd)
        ref, tol = reference(x3, hs3, oh3, dh3, adjoint, dt)
        err = np.abs(y3.reshape(ref.shape).astype(np.float64) - y2.reshape(ref.shape).astype(np.float64))
        assert np.all(err <= 2 * tol), f"max diff {err.max():.3e}"
        check_close(y3, x3, hs3, oh3, dh3, adjoint, dt)


@pytest.mark.gpu
def test_kernel_error_codes_leave_y_untouched(pm):
    import torch
    L = pm._lib
    x = torch.arange(48, dtype=torch.float64, device="cuda")
    y = torch.full((48,), 3.5, dtype=torch.float64, device="cuda")
    hs = torch.ones(2 * 2 * 2 * 3 * 3 * 3, dtype=torch.float64, device="cuda")
    ARG, DT = 2002, 2001
    cases = [
        (dict(x=None), ARG), (dict(y=None), ARG), (dict(hs=None), ARG), (dict(y="x"), ARG),
        (dict(dims=(0, 3, 2)), ARG), (dict(dims=(4, 0, 2)), ARG), (dict(dims=(4, 3, 0)), ARG),
        (dict(ni=0), ARG), (dict(ni=3), ARG),
        (dict(nf=(0, 2, 2)), ARG), (dict(nf=(2, 0, 2)), ARG), (dict(nf=(2, 2, -1)), ARG),
        (dict(nh=(0, 3, 3)), ARG), (dict(nh=(3, -1, 3)), ARG), (dict(nh=(3, 3, 0)), ARG),
        (dict(dh=(0, 1, 1)), ARG), (dict(dh=(1, -2, 1)), ARG), (dict(dh=(1, 1, 0)), ARG),
        (dict(dims=(4, 3, 2 ** 29)), ARG), (dict(dh=(2 ** 29, 1, 1)), ARG),     # past the kernel's 32-bit axes
        (dict(dtype=L.C64), DT), (dict(dtype=L.C128), DT), (dict(dtype=L.BF16), DT), (dict(dtype=99), DT),
    ]
    assert_rejected(lambda a: c_ns(pm, a["x"], a["y"], a["dims"], a["ni"], a["hs"], a["nf"], a["nh"], (0, 0, 0), a["dh"],
                                   0, a["dtype"]),
                    dict(x=x.data_ptr(), y=y.data_ptr(), hs=hs.data_ptr(), dims=(4, 3, 2), ni=2, nf=(2, 2, 2),
                         nh=(3, 3, 3), dh=(2, 1, 1), dtype=L.F64), cases, y)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the operator
# ---------------------------------------------------------------------------------------------------------------
def local_ops(pm, nh, bank, dt):
    hs, ih, _, _ = mg3.case_inputs(nh, bank, dt)
    return [pm.local.NonStationaryConvolve3D((mg3.NX, mg3.NY, mg3.NZ), hs[k], *ih, dtype=hs.dtype)
            for k in range(mg3.NV)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", mg3.cases(), ids=[case_id(c) for c in mg3.cases()])
def test_operator_vs_reference_fixtures(pm, case):
    nh, bank, dt = case
    _, _, x, v = mg3.case_inputs(nh, bank, dt)
    Op = pm.MPIBlockDiag(local_ops(pm, nh, bank, dt), dtype=dt)
    got = host((Op @ pm.DistributedArray.to_dist(x)).asarray())
    gota = host((Op.H @ pm.DistributedArray.to_dist(v)).asarray())
    assert got.dtype == np.dtype(dt) and gota.dtype == np.dtype(dt)
    gy, gya = decode(GOLD, mg3.key(nh, bank), dt, mg3.ENC)
    np.testing.assert_array_equal(got, gy)
    np.testing.assert_array_equal(gota, gya)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["float64", "float32", "complex128"])
def test_operator_dottest(pm, dt):
    from pylops_mpi_b200.utils.dottest import dottest
    rng = np.random.default_rng(8)
    rdt = "float32" if dt == "float32" else "float64"
    ops = [pm.local.NonStationaryConvolve3D((13, 21, 17), rng.standard_normal((3, 2, 3, 5, 7, 3)).astype(rdt),
                                            [2, 6, 10], [3, 13], [1, 8, 15], dtype=rdt) for _ in range(3)]
    Op = pm.MPIBlockDiag(ops, dtype=dt)
    n = Op.shape[0]
    u = rng.standard_normal(n) + (1j * rng.standard_normal(n) if dt == "complex128" else 0)
    v = rng.standard_normal(n) + (1j * rng.standard_normal(n) if dt == "complex128" else 0)
    assert dottest(Op, pm.DistributedArray.to_dist(u.astype(dt)), pm.DistributedArray.to_dist(v.astype(dt)),
                   rtol=1e-5 if dt == "float32" else 1e-12)


@pytest.mark.gpu
def test_operator_attributes_dtypes_and_out(pm):
    import torch
    rng = np.random.default_rng(4)
    hs = rng.standard_normal((3, 2, 2, 5, 3, 7))
    dims, N = (12, 7, 9), 12 * 7 * 9
    Op = pm.local.NonStationaryConvolve3D(dims, hs.astype(np.float32), [2, 6, 10], [1, 4], [0, 5], dtype="float32",
                                          engine="cuda", num_threads_per_blocks=(4, 8, 8))
    assert Op.dims == Op.dimsd == dims and Op.shape == (N, N) and Op.dtype == np.float32
    assert (Op.nfilt, Op.nh, Op.hc, Op.oh, Op.dh) == ((3, 2, 2), (5, 3, 7), (2, 1, 3), (2, 1, 0), (4, 3, 5))
    assert pm.local.NonStationaryConvolve3D(dims, hs[:1, :1, :1], [7], [0], [3]).dh == (1, 1, 1)
    # float32 data of a float64-bank float32 operator: the bank rounded to float32
    M = ns_matrix(hs.astype(np.float32), dims, (2, 1, 0), (4, 3, 5))
    x = rng.standard_normal(N).astype(np.float32)
    y = host(Op.matvec(torch.as_tensor(x).cuda()))
    np.testing.assert_allclose(y, M @ x, rtol=0, atol=1e-4 * np.abs(M).sum(1).max())


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["float32", "float64"])
def test_cgls_graph_replay_matches_step_loop(pm, dt):
    rng = np.random.default_rng(12)
    hs = rng.standard_normal((3, 2, 3, 5, 7, 3)).astype(dt)
    Op = pm.MPIBlockDiag([pm.local.NonStationaryConvolve3D((14, 20, 15), hs, [2, 7, 12], [3, 13], [1, 7, 13],
                                                           dtype=dt) for _ in range(2)])
    n = Op.shape[0]
    y = Op @ pm.DistributedArray.to_dist(rng.standard_normal(n).astype(dt))
    assert_cgls_replay_matches_steps(pm, Op, y, pm.DistributedArray.to_dist(np.zeros(n, dtype=dt)), 25, 20)


@pytest.mark.gpu
def test_flow_psfs_from_device_kirchhoff(pm):
    """the point-spread functions of the device 3-D local.Kirchhoff (K^H K of the point scatterers) are the stored
    ones"""
    import torch
    z, x, t, srcs, recs, vel, wav, wavc, y = mg3.flow_geometry()
    K = pm.local.Kirchhoff(z, x, t, srcs, recs, vel, wav, wavc, y=y, mode="analytic")
    m_psf, m_true = mg3.flow_models()
    img = host(K.rmatvec(K.matvec(torch.as_tensor(m_psf.ravel()).cuda())))
    hs = mg3.psf_windows(img.reshape(mg3.FLOW_NY, mg3.FLOW_NX, mg3.FLOW_NZ))
    scale = np.abs(GOLD["flow/hs"]).max()
    np.testing.assert_allclose(hs, GOLD["flow/hs"], rtol=0, atol=1e-12 * scale)
    mmig = np.concatenate([host(K.rmatvec(K.matvec(torch.as_tensor(m.ravel()).cuda()))) for m in m_true])
    np.testing.assert_allclose(mmig, GOLD["flow/mmig"], rtol=0, atol=1e-12 * np.abs(GOLD["flow/mmig"]).max())


def flow_tolerance():
    """(x, cost) relative tolerances of the flow: the cgls run summed in another order than pylops' moves by about
    what a 4-ulp jitter of every apply moves the reference's own run (``flow/spread``), and by no less than
    cond * 2^-53 (``flow/cond``, about 6e6, the PSF operator's condition number); the test allows 100 and 10 times
    those"""
    floor = 10 * float(GOLD["flow/cond"]) * 2.0 ** -53
    return tuple(max(100 * float(s), floor) for s in GOLD["flow/spread"])


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
def test_image_domain_lsm_flow_vs_reference(pm, P):
    """cgls on MPIBlockDiag([NonStationaryConvolve3D(psfs)] * nv_r) from the stored bank and migrated volumes: the
    blocks of P ranks' volumes as one rank's blocks"""
    ops = [pm.local.NonStationaryConvolve3D((mg3.FLOW_NY, mg3.FLOW_NX, mg3.FLOW_NZ), GOLD["flow/hs"], mg3.FLOW_IHY,
                                            mg3.FLOW_IHX, mg3.FLOW_IHZ)
           for nv in rows_of(P, mg3.FLOW_NV) for _ in range(nv)]
    Op = pm.MPIBlockDiag(ops)
    d = pm.DistributedArray.to_dist(GOLD["flow/mmig"])
    x0 = pm.DistributedArray.to_dist(np.zeros_like(GOLD["flow/mmig"]))
    x, _, iiter, _, _, cost = pm.cgls(Op, d, x0=x0, niter=mg3.FLOW_NITER, tol=0.0)
    assert iiter == int(GOLD[f"flow/P{P}/iiter"])
    xtol, ctol = flow_tolerance()
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"flow/P{P}/cost"], rtol=ctol)
    gx = GOLD[f"flow/P{P}/x"]
    np.testing.assert_allclose(host(x.asarray()), gx, rtol=0, atol=xtol * np.abs(gx).max())


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [1, 2])
def test_multi_rank_fixtures(nproc):
    needs_gpus(nproc)
    run_on_ranks("test_nsconvolve3d", nproc)


def on_ranks(pm, comm):
    """each rank's MPIBlockDiag block of NonStationaryConvolve3D against its slice of the gathered fixtures, and
    the 3-D image-domain cgls flow against its fixture"""
    rank, P = comm.Get_rank(), comm.Get_size()
    def block(nv_global, volume):
        """this rank's volumes of a (nv_global, ...) stack: (local_shapes, flat slice, first volume, volume count)"""
        rows = rows_of(P, nv_global)
        k0 = sum(rows[:rank])
        return [(r * volume,) for r in rows], slice(k0 * volume, (k0 + rows[rank]) * volume), k0, rows[rank]

    ls, sl, k0, nv = block(mg3.NV, mg3.NX * mg3.NY * mg3.NZ)
    for nh, bank, dt in mg3.cases():
        hs, ih, x, v = mg3.case_inputs(nh, bank, dt)
        Op = pm.MPIBlockDiag([pm.local.NonStationaryConvolve3D((mg3.NX, mg3.NY, mg3.NZ), hs[k], *ih, dtype=hs.dtype)
                              for k in range(k0, k0 + nv)], dtype=dt)
        gy, gya = decode(GOLD, mg3.key(nh, bank), dt, mg3.ENC)
        name = f"{mg3.key(nh, bank)}/{dt}"
        np.testing.assert_array_equal(host((Op @ pm.DistributedArray.to_dist(x, local_shapes=ls)).local_array), gy[sl],
                                      err_msg=f"[rank {rank}] {name}/y")
        np.testing.assert_array_equal(host((Op.H @ pm.DistributedArray.to_dist(v, local_shapes=ls)).local_array),
                                      gya[sl], err_msg=f"[rank {rank}] {name}/ya")

    ls, sl, k0, nv = block(mg3.FLOW_NV, mg3.FLOW_NY * mg3.FLOW_NX * mg3.FLOW_NZ)
    Op = pm.MPIBlockDiag([pm.local.NonStationaryConvolve3D((mg3.FLOW_NY, mg3.FLOW_NX, mg3.FLOW_NZ), GOLD["flow/hs"],
                                                           mg3.FLOW_IHY, mg3.FLOW_IHX, mg3.FLOW_IHZ)] * nv)
    mmig = GOLD["flow/mmig"]
    d = pm.DistributedArray.to_dist(mmig, local_shapes=ls)
    x0 = pm.DistributedArray.to_dist(np.zeros_like(mmig), local_shapes=ls)
    x, _, iiter, _, _, cost = pm.cgls(Op, d, x0=x0, niter=mg3.FLOW_NITER, tol=0.0)
    assert iiter == int(GOLD[f"flow/P{P}/iiter"])
    xtol, ctol = flow_tolerance()
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"flow/P{P}/cost"], rtol=ctol, err_msg=f"[rank {rank}] cost")
    gx = GOLD[f"flow/P{P}/x"]
    np.testing.assert_allclose(host(x.local_array), gx[sl], rtol=0, atol=xtol * np.abs(gx).max(),
                               err_msg=f"[rank {rank}] x")
