"""Rank-local NonStationaryConvolve2D (pylops.signalprocessing inside MPIBlockDiag) and image-domain least-squares
migration with point-spread functions.

    h_j = sum_(a,b) T(wx_a(jx) wz_b(jz)) hs[a, b]     bilinear in the bank (end filters outside the nodes)
    forward y[i] = sum_j h_j[hc + i - j] x[j],  adjoint the transpose

CPU: refshim's restatement against that definition, the interpolation weights, the operator's argument errors, and
the fixtures of tests/golden/nsconvolve2d_golden.npz (made by make_golden_nsconvolve2d.py: the reference's
MPIBlockDiag and cgls over the restatement; operator inputs exactly representable, so every dtype must match them
bit for bit).  GPU: b2_nsconvolve2d through the C ABI, and the operator through the public interface."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_nsconvolve2d as mg2  # noqa: E402
from ns_reference import axis_weights, c_ns, check_close, ns_matrix, point_weights, run_kernel  # noqa: E402
from fixture_codec import decode, rows_of  # noqa: E402
from op_checks import assert_cgls_replay_matches_steps, assert_rejected, host, needs_gpus, run_on_ranks  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "nsconvolve2d_golden.npz"), allow_pickle=False)


def refshim():
    path = os.path.join(HERE, "golden", "refshim")
    sys.path.insert(0, path)
    try:
        from pylops.signalprocessing.nonstatconvolve2d import NonStationaryConvolve2D
    finally:
        sys.path.remove(path)
    return NonStationaryConvolve2D


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nh", [(1, 1), (3, 5), (7, 3)])
@pytest.mark.parametrize("nf,dh,oh", [((1, 1), (1, 1), (0, 3)), ((2, 3), (3, 2), (1, 2)), ((3, 2), (4, 5), (2, 0))])
def test_refshim_restatement_is_the_definition(nh, nf, dh, oh):
    NS2 = refshim()
    rng = np.random.default_rng(nh[0] * 10 + nh[1] + nf[0])
    hs = rng.standard_normal(nf + nh)
    ihx, ihz = oh[0] + dh[0] * np.arange(nf[0]), oh[1] + dh[1] * np.arange(nf[1])
    dims = (11, 13)
    Op = NS2(dims, hs, ihx, ihz)
    M = ns_matrix(hs, dims, oh, dh)
    x = rng.standard_normal(dims[0] * dims[1])
    np.testing.assert_allclose(Op.matvec(x), M @ x, rtol=0, atol=1e-12)
    np.testing.assert_allclose(Op.rmatvec(x), M.T @ x, rtol=0, atol=1e-12)


@pytest.mark.parametrize("nf,dh,oh", [(1, 1, 0), (1, 1, 5), (2, 3, 1), (4, 4, 2), (5, 7, 6)])
def test_interpolation_weights_and_clamps(nf, dh, oh):
    NS2 = refshim()
    for j in range(40):
        l, r, wl, wr = NS2.weights(j, oh, dh, nf)
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
    # the interpolated filter: pylops' four-term sum equals the definition within float64 rounding
    rng = np.random.default_rng(nf)
    hs = rng.standard_normal((nf, 3, 5, 3))
    Op = NS2((40, 12), hs, oh + dh * np.arange(nf), [1, 5, 9])
    for jx in range(0, 40, 3):
        for jz in range(12):
            want = sum(W * hs[a, b] for (a, b), W in point_weights((jx, jz), (oh, 1), (dh, 4), (nf, 3), np.float64))
            np.testing.assert_allclose(Op.interpolate_h(jx, jz), want, rtol=0, atol=1e-15)


def test_operator_argument_errors():
    import pylops_mpi_b200.local as L
    NSC = L.NonStationaryConvolve2D
    hs = np.ones((3, 2, 5, 3))
    good = dict(dims=(20, 10), hs=hs, ihx=[2, 6, 10], ihz=[1, 4])
    for bad in (dict(hs=np.ones((3, 2, 4, 3))), dict(hs=np.ones((3, 2, 5, 2))),      # even filter sizes
                dict(ihx=[2, 6, 11]), dict(ihz=[1, 4, 8]),                          # irregular, wrong count
                dict(ihx=[2, 6]),                                                   # len(ihx) != nfx
                dict(ihx=[-1, 3, 7]), dict(ihx=[10, 15, 20]), dict(ihz=[5, 10]),    # outside [0, dims)
                dict(ihx=[10, 6, 2]), dict(ihz=[4, 1]),                             # decreasing
                dict(hs=np.ones((3, 5, 3))), dict(dims=(20, 10, 1)), dict(dims=(200,))):
        kw = dict(good)
        kw.update(bad)
        with pytest.raises(ValueError):
            NSC(kw["dims"], kw["hs"], kw["ihx"], kw["ihz"])
    with pytest.raises(NotImplementedError):
        NSC((20, 10), hs + 1j, [2, 6, 10], [1, 4])


def test_fixture_inventory():
    want = set()
    for nh, bank, dt in mg2.cases():
        k = mg2.key(nh, bank)
        for n in ("y", "ya", "yi", "yai")[:4 if dt == "complex128" else 2]:
            assert GOLD[f"{k}/{n}"].dtype == np.int32 and GOLD[f"{k}/{n}"].shape == (mg2.NY * mg2.NX * mg2.NZ,)
            want.add(f"{k}/{n}")
    assert len(want) == 2 * len(mg2.NHS) * len(mg2.BANKS) + 2 * 2
    flows = {f"flow/P{P}/{k}" for P in (1, 2, 3) for k in ("x", "iiter", "cost")}
    assert sorted(GOLD.files) == sorted(want | flows | {"flow/hs", "flow/mmig"})
    assert max(nh[0] for nh in mg2.NHS) >= 41 and any(nh[0] != nh[1] for nh in mg2.NHS)
    for P in (1, 2, 3):
        assert int(GOLD[f"flow/P{P}/iiter"]) == mg2.FLOW_NITER


def case_id(c):
    nh, ((nfx, nfz), (dhx, dhz)), dt = c
    return f"nh{nh[0]}x{nh[1]}/nf{nfx}x{nfz}/dh{dhx}x{dhz}/{dt}"


def slices(a):
    n = mg2.NX * mg2.NZ
    return [a[k * n:(k + 1) * n] for k in range(mg2.NY)]


@pytest.mark.parametrize("case", mg2.cases(), ids=[case_id(c) for c in mg2.cases()])
def test_fixtures_follow_the_restatement_in_every_dtype(case):
    NS2 = refshim()
    nh, bank, dt = case
    hs, ihx, ihz, x, v = mg2.case_inputs(nh, bank, dt)
    ops = [NS2((mg2.NX, mg2.NZ), hs[k], ihx, ihz, dtype=dt) for k in range(mg2.NY)]
    y = np.concatenate([op.matvec(s) for op, s in zip(ops, slices(x))])
    ya = np.concatenate([op.rmatvec(s) for op, s in zip(ops, slices(v))])
    gy, gya = decode(GOLD, mg2.key(nh, bank), dt, mg2.ENC)
    assert y.dtype == np.dtype(dt) and gy.dtype == np.dtype(dt)
    np.testing.assert_array_equal(y, gy)
    np.testing.assert_array_equal(ya, gya)
    if dt != "complex128":          # the other real dtype gives the same values (the generator checks all three)
        other = decode(GOLD, mg2.key(nh, bank), "float32" if dt == "float64" else "float64", mg2.ENC)
        np.testing.assert_array_equal(gy.astype(np.float64), other[0].astype(np.float64))


def test_flow_psfs_follow_the_restated_kirchhoff():
    kirchhoff, _ = mg2.refshim_kirchhoff()
    K = kirchhoff.Kirchhoff(*mg2.flow_geometry(), mode="analytic")
    m_psf, m_true = mg2.flow_models()
    img = K.rmatvec(K.matvec(m_psf.ravel())).reshape(mg2.FLOW_NX, mg2.FLOW_NZ)
    np.testing.assert_array_equal(mg2.psf_windows(img), GOLD["flow/hs"])
    np.testing.assert_array_equal(K.rmatvec(K.matvec(m_true[1].ravel())),
                                  GOLD["flow/mmig"][mg2.FLOW_NX * mg2.FLOW_NZ:2 * mg2.FLOW_NX * mg2.FLOW_NZ])


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernel through the C ABI
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


SHAPES = [(1, 1), (1, 37), (29, 1), (5, 7), (33, 65), (70, 130)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("nh", [(1, 1), (3, 5), (9, 7), (41, 41)], ids=lambda v: f"nh{v[0]}x{v[1]}")
def test_kernel_vs_matrix(pm, dt, nh):
    rng = np.random.default_rng(nh[0] * 100 + nh[1])
    for dims in SHAPES:
        for nf, dh, oh in (((1, 1), (1, 1), (0, 0)), ((2, 3), (3, 4), (0, 1)), ((3, 2), (5, 7), (2, 3)),
                           ((2, 2), (1, 1), (0, 0))):
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
@pytest.mark.parametrize("case", ["129x129/small", "129x129/steps", "65x129/wide", "127x3/tall"])
def test_kernel_large_filters_in_chunks(pm, dt, case):
    """filters larger than one chunk of taps, images smaller than the filter, steps that do not divide dims"""
    nh, dims, nf, dh = {"129x129/small": ((129, 129), (20, 30), (1, 1), (1, 1)),
                        "129x129/steps": ((129, 129), (37, 41), (3, 4), (13, 9)),
                        "65x129/wide": ((65, 129), (40, 150), (2, 5), (30, 31)),
                        "127x3/tall": ((127, 3), (160, 9), (6, 2), (31, 7))}[case]
    rng = np.random.default_rng(len(case))
    hs = rng.standard_normal(nf + nh).astype(dt)
    x = rng.standard_normal(dims + (1,)).astype(dt)
    for adjoint in (False, True):
        y, guards, same = run_kernel(pm, x, hs, (1, 2), dh, adjoint, dt)
        assert guards and same
        check_close(y, x, hs, (1, 2), dh, adjoint, dt)


@pytest.mark.gpu
def test_kernel_error_codes_leave_y_untouched(pm):
    import torch
    L = pm._lib
    x = torch.arange(24, dtype=torch.float64, device="cuda")
    y = torch.full((24,), 3.5, dtype=torch.float64, device="cuda")
    hs = torch.ones(2 * 2 * 3 * 3, dtype=torch.float64, device="cuda")
    ARG, DT = 2002, 2001
    cases = [
        (dict(x=None), ARG), (dict(y=None), ARG), (dict(hs=None), ARG), (dict(y="x"), ARG),
        (dict(nx=0), ARG), (dict(nz=0), ARG), (dict(ni=0), ARG), (dict(ni=3), ARG),
        (dict(nf=(0, 2)), ARG), (dict(nf=(2, 0)), ARG), (dict(nh=(0, 3)), ARG), (dict(nh=(3, -1)), ARG),
        (dict(dh=(0, 1)), ARG), (dict(dh=(1, -2)), ARG),
        (dict(dtype=L.C64), DT), (dict(dtype=L.C128), DT), (dict(dtype=L.BF16), DT), (dict(dtype=99), DT),
    ]
    assert_rejected(lambda a: c_ns(pm, a["x"], a["y"], (a["nx"], a["nz"]), a["ni"], a["hs"], a["nf"], a["nh"], (0, 0),
                                   a["dh"], 0, a["dtype"]),
                    dict(x=x.data_ptr(), y=y.data_ptr(), hs=hs.data_ptr(), nx=4, nz=3, ni=2, nf=(2, 2), nh=(3, 3),
                         dh=(2, 1), dtype=L.F64), cases, y)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the operator
# ---------------------------------------------------------------------------------------------------------------
def local_ops(pm, nh, bank, dt):
    hs, ihx, ihz, _, _ = mg2.case_inputs(nh, bank, dt)
    return [pm.local.NonStationaryConvolve2D((mg2.NX, mg2.NZ), hs[k], ihx, ihz, dtype=hs.dtype)
            for k in range(mg2.NY)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", mg2.cases(), ids=[case_id(c) for c in mg2.cases()])
def test_operator_vs_reference_fixtures(pm, case):
    nh, bank, dt = case
    _, _, _, x, v = mg2.case_inputs(nh, bank, dt)
    Op = pm.MPIBlockDiag(local_ops(pm, nh, bank, dt), dtype=dt)
    got = host((Op @ pm.DistributedArray.to_dist(x)).asarray())
    gota = host((Op.H @ pm.DistributedArray.to_dist(v)).asarray())
    assert got.dtype == np.dtype(dt) and gota.dtype == np.dtype(dt)
    gy, gya = decode(GOLD, mg2.key(nh, bank), dt, mg2.ENC)
    np.testing.assert_array_equal(got, gy)
    np.testing.assert_array_equal(gota, gya)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["float64", "float32", "complex128"])
def test_operator_dottest(pm, dt):
    from pylops_mpi_b200.utils.dottest import dottest
    rng = np.random.default_rng(8)
    rdt = "float32" if dt == "float32" else "float64"
    ops = [pm.local.NonStationaryConvolve2D((31, 47), rng.standard_normal((3, 4, 7, 11)).astype(rdt), [2, 12, 22],
                                            [3, 13, 23, 33], dtype=rdt) for _ in range(3)]
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
    hs = rng.standard_normal((3, 2, 5, 7))
    Op = pm.local.NonStationaryConvolve2D((20, 9), hs.astype(np.float32), [2, 6, 10], [1, 4], dtype="float32",
                                          engine="cuda", num_threads_per_blocks=(8, 8))
    assert Op.dims == (20, 9) and Op.shape == (180, 180) and Op.dtype == np.float32
    assert (Op.nfilt, Op.nh, Op.hc, Op.oh, Op.dh) == ((3, 2), (5, 7), (2, 3), (2, 1), (4, 3))
    assert pm.local.NonStationaryConvolve2D((20, 9), hs[:1, :1], [7], [0]).dh == (1, 1)
    # float32 data of a float64-bank float32 operator: the bank rounded to float32
    M = ns_matrix(hs.astype(np.float32), (20, 9), (2, 1), (4, 3))
    x = rng.standard_normal(180).astype(np.float32)
    y = host(Op.matvec(torch.as_tensor(x).cuda()))
    np.testing.assert_allclose(y, M @ x, rtol=0, atol=1e-4 * np.abs(M).sum(1).max())


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["float32", "float64"])
def test_cgls_graph_replay_matches_step_loop(pm, dt):
    rng = np.random.default_rng(12)
    hs = rng.standard_normal((4, 3, 9, 7)).astype(dt)
    Op = pm.MPIBlockDiag([pm.local.NonStationaryConvolve2D((40, 30), hs, [3, 13, 23, 33], [2, 12, 22], dtype=dt)
                          for _ in range(2)])
    n = Op.shape[0]
    y = Op @ pm.DistributedArray.to_dist(rng.standard_normal(n).astype(dt))
    assert_cgls_replay_matches_steps(pm, Op, y, pm.DistributedArray.to_dist(np.zeros(n, dtype=dt)), 25, 20)


@pytest.mark.gpu
def test_flow_psfs_from_device_kirchhoff(pm):
    """the point-spread functions of local.Kirchhoff (K^H K of the point scatterers) are the stored ones"""
    import torch
    K = pm.local.Kirchhoff(*mg2.flow_geometry(), mode="analytic")
    m_psf, m_true = mg2.flow_models()
    img = host(K.rmatvec(K.matvec(torch.as_tensor(m_psf.ravel()).cuda()))).reshape(mg2.FLOW_NX, mg2.FLOW_NZ)
    hs = mg2.psf_windows(img)
    scale = np.abs(GOLD["flow/hs"]).max()
    np.testing.assert_allclose(hs, GOLD["flow/hs"], rtol=0, atol=1e-12 * scale)
    mmig = np.concatenate([host(K.rmatvec(K.matvec(torch.as_tensor(m.ravel()).cuda()))) for m in m_true])
    np.testing.assert_allclose(mmig, GOLD["flow/mmig"], rtol=0, atol=1e-12 * np.abs(GOLD["flow/mmig"]).max())


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
def test_image_domain_lsm_flow_vs_reference(pm, P):
    """cgls on MPIBlockDiag([NonStationaryConvolve2D(psfs)] * ny_r) from the stored bank and migrated images: the
    blocks of P ranks' rows as one rank's blocks.  The PSF operator's condition number is about 2e6, so 20 iterations
    summed in another order than pylops' may move x by about cond * 2^-53 ~ 2e-10 of max |x|"""
    ops = [pm.local.NonStationaryConvolve2D((mg2.FLOW_NX, mg2.FLOW_NZ), GOLD["flow/hs"], mg2.FLOW_IHX, mg2.FLOW_IHZ)
           for ny in rows_of(P, mg2.FLOW_NY) for _ in range(ny)]
    Op = pm.MPIBlockDiag(ops)
    d = pm.DistributedArray.to_dist(GOLD["flow/mmig"])
    x0 = pm.DistributedArray.to_dist(np.zeros_like(GOLD["flow/mmig"]))
    x, _, iiter, _, _, cost = pm.cgls(Op, d, x0=x0, niter=mg2.FLOW_NITER, tol=0.0)
    assert iiter == int(GOLD[f"flow/P{P}/iiter"])
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"flow/P{P}/cost"], rtol=1e-10)
    gx = GOLD[f"flow/P{P}/x"]
    np.testing.assert_allclose(host(x.asarray()), gx, rtol=1e-9, atol=1e-10 * np.abs(gx).max())


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [1, 2])
def test_multi_rank_fixtures(nproc):
    needs_gpus(nproc)
    run_on_ranks("test_nsconvolve2d", nproc)


def on_ranks(pm, comm):
    """each rank's MPIBlockDiag block of NonStationaryConvolve2D against its slice of the gathered fixtures, and
    the image-domain cgls flow against its fixture"""
    rank, P = comm.Get_rank(), comm.Get_size()
    def block(ny_global, plane):
        """this rank's slices of a (ny_global, ...) stack: (local_shapes, flat slice, first slice, slice count)"""
        rows = rows_of(P, ny_global)
        k0 = sum(rows[:rank])
        return [(r * plane,) for r in rows], slice(k0 * plane, (k0 + rows[rank]) * plane), k0, rows[rank]

    ls, sl, k0, ny = block(mg2.NY, mg2.NX * mg2.NZ)
    for nh, bank, dt in mg2.cases():
        hs, ihx, ihz, x, v = mg2.case_inputs(nh, bank, dt)
        Op = pm.MPIBlockDiag([pm.local.NonStationaryConvolve2D((mg2.NX, mg2.NZ), hs[k], ihx, ihz, dtype=hs.dtype)
                              for k in range(k0, k0 + ny)], dtype=dt)
        gy, gya = decode(GOLD, mg2.key(nh, bank), dt, mg2.ENC)
        name = f"{mg2.key(nh, bank)}/{dt}"
        np.testing.assert_array_equal(host((Op @ pm.DistributedArray.to_dist(x, local_shapes=ls)).local_array), gy[sl],
                                      err_msg=f"[rank {rank}] {name}/y")
        np.testing.assert_array_equal(host((Op.H @ pm.DistributedArray.to_dist(v, local_shapes=ls)).local_array),
                                      gya[sl], err_msg=f"[rank {rank}] {name}/ya")

    ls, sl, k0, ny = block(mg2.FLOW_NY, mg2.FLOW_NX * mg2.FLOW_NZ)
    Op = pm.MPIBlockDiag([pm.local.NonStationaryConvolve2D((mg2.FLOW_NX, mg2.FLOW_NZ), GOLD["flow/hs"], mg2.FLOW_IHX,
                                                           mg2.FLOW_IHZ)] * ny)
    mmig = GOLD["flow/mmig"]
    d = pm.DistributedArray.to_dist(mmig, local_shapes=ls)
    x0 = pm.DistributedArray.to_dist(np.zeros_like(mmig), local_shapes=ls)
    x, _, iiter, _, _, cost = pm.cgls(Op, d, x0=x0, niter=mg2.FLOW_NITER, tol=0.0)
    assert iiter == int(GOLD[f"flow/P{P}/iiter"])
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"flow/P{P}/cost"], rtol=1e-10, err_msg=f"[rank {rank}] cost")
    gx = GOLD[f"flow/P{P}/x"]
    np.testing.assert_allclose(host(x.local_array), gx[sl], rtol=1e-9, atol=1e-10 * np.abs(gx).max(),
                               err_msg=f"[rank {rank}] x")
