"""GPU parity tests, operator level (world_size 1): the reference-facing API
(DistributedArray, MPI* operators, dottest, cgls) against the CPU oracle and
the reference's own known-answer vectors.  Multi-rank runs of the same checks
live in tests/test_gpu_multi.py (needs >= 2 GPUs)."""
import numpy as np
import pytest
import torch

import pylops_mpi_oracle as o
from op_checks import host

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


# ---- DistributedArray: test_distributedarray.py ------------------------------------------
@pytest.mark.parametrize("shape,axis", [((500, 501), 1), ((501, 500), 0), ((200, 31, 11), 1), ((600,), 0)])
@pytest.mark.parametrize("dtype", [np.float64, np.complex128, np.float32])
def test_creation_to_dist_math(pm, shape, axis, dtype):
    np.random.seed(42)
    a = np.random.normal(100, 100, shape).astype(dtype)
    b = np.random.normal(300, 300, shape).astype(dtype)
    if np.issubdtype(dtype, np.complexfloating):
        a = a + 1j * np.random.normal(0, 50, shape)
        b = b - 1j * np.random.normal(0, 50, shape)
    A = pm.DistributedArray.to_dist(a, axis=axis)
    B = pm.DistributedArray.to_dist(b, axis=axis)
    assert A.global_shape == shape and A.local_shape == shape and A.local_shapes == [shape]
    assert A.partition is pm.Partition.SCATTER and A.axis == axis and A.dtype == np.dtype(dtype)
    tol = dict(rtol=1e-5) if dtype == np.float32 else dict(rtol=1e-14)
    np.testing.assert_allclose(host((A + B).asarray()), a + b, **tol)
    np.testing.assert_allclose(host((A - B).asarray()), a - b, **tol)
    np.testing.assert_allclose(host((A * B).asarray()), a * b, **tol)
    np.testing.assert_allclose(host((A * 3.5).asarray()), a * 3.5, **tol)
    np.testing.assert_allclose(host((2 * A).asarray()), 2 * a, **tol)
    np.testing.assert_allclose(host((-A).asarray()), -a, **tol)
    np.testing.assert_allclose(host(A.conj().asarray()), a.conj(), **tol)
    Cc = A.copy()
    Cc += B
    Cc -= A
    if dtype == np.float32:   # (a + b) - a carries one ulp of |a + b|
        np.testing.assert_allclose(host(Cc.asarray()), b, rtol=1e-4, atol=1e-3)
    else:
        np.testing.assert_allclose(host(Cc.asarray()), b, rtol=1e-12)
    assert np.all(host(A.zeros_like().asarray()) == 0)
    r = A.ravel()
    assert r.global_shape == (int(np.prod(shape)),)
    np.testing.assert_array_equal(host(r.asarray()), a.ravel())
    # dot / norm (test_distributedarray.py:201-222)
    scale = np.linalg.norm(a) * np.linalg.norm(b)
    rt = 1e-5 if dtype == np.float32 else 1e-13
    assert abs(A.dot(B)[0] - np.dot(a.ravel().astype(np.complex128), b.ravel().astype(np.complex128))) <= rt * scale
    assert abs(A.dot(B, vdot=True)[0] - np.vdot(a.ravel().astype(np.complex128), b.ravel().astype(np.complex128))) <= rt * scale
    for ord_ in (None, 1, 2, np.inf, -np.inf, 0, 3):
        ref = np.linalg.norm(a.ravel().astype(np.complex128), 2 if ord_ is None else ord_)
        got = A.norm(ord_)
        assert got.dtype == np.float64 and got.shape == (1,)
        np.testing.assert_allclose(got[0], ref, rtol=rt)


def test_broadcast_and_errors(pm):
    x = np.arange(12.0).reshape(3, 4)
    B = pm.DistributedArray.to_dist(x, partition=pm.Partition.BROADCAST)
    assert B.local_shape == (3, 4)
    np.testing.assert_allclose(B.dot(B)[0], (x * x).sum())
    np.testing.assert_allclose(B.norm()[0], np.linalg.norm(x))
    with pytest.raises(IndexError):
        pm.DistributedArray(global_shape=(3,), axis=1)
    with pytest.raises(ValueError):
        pm.DistributedArray(global_shape=(3,), local_shapes=[(2,)])
    S = pm.DistributedArray.to_dist(x)
    with pytest.raises(ValueError):
        S + B
    with pytest.raises(ValueError):
        S.add(pm.DistributedArray.to_dist(np.zeros((3, 5))))
    g = S.add_ghost_cells(cells_front=1, cells_back=1)
    np.testing.assert_array_equal(host(g), x)
    assert S.redistribute(1).axis == 1


# ---- MPIFirstDerivative: config 1 and the test_derivative.py grid ----------------------------
def test_config1_readme_flow(pm):
    """README.md:73-94 / plot_derivative.py:36-43 + dottest + cgls(niter=10)"""
    nz, nx = 11, 21
    x = np.zeros((nz, nx))
    x[nz // 2, nx // 2] = 1.0
    xd = pm.DistributedArray.to_dist(x.ravel())
    Fop = pm.MPIFirstDerivative((nz, nx), dtype=np.float64)
    y = Fop @ xd
    yh = host(y.asarray()).reshape(nz, nx)
    expect = np.zeros((nz, nx))
    expect[4, 10], expect[6, 10] = 0.5, -0.5
    assert np.array_equal(yh, expect)
    # the oracle at P=2 (the reference's run) gives the same global answer
    ref = np.concatenate(o.first_derivative(o.to_dist(x.ravel(), 2), (nz, nx)))
    assert np.array_equal(yh.ravel(), ref)
    u = pm.DistributedArray.to_dist(np.random.default_rng(42).normal(0, 10, nz * nx))
    v = pm.DistributedArray.to_dist(np.random.default_rng(43).normal(0, 10, nz * nx))
    assert pm.dottest(Fop, u, v, rtol=1e-6)
    # cgls 10 iterations vs the oracle (P=2 simulation of the reference)
    x0 = pm.DistributedArray.to_dist(np.zeros(nz * nx))
    xinv, istop, iit, r1, r2, cost = pm.cgls(Fop, y, x0=x0, niter=10, tol=0.0)
    mv = lambda a: o.SimArray(o.first_derivative(a.locs, (nz, nx)))                  # noqa: E731
    rmv = lambda a: o.SimArray(o.first_derivative(a.locs, (nz, nx), adjoint=True))   # noqa: E731
    yo = mv(o.SimArray(o.to_dist(x.ravel(), 2)))
    # the operator's outputs live on the row-block partition [126, 105]; the reference's cgls
    # needs x0 on that same partition (DistributedArray._check_partition_shape)
    x0o = o.SimArray([np.zeros(126), np.zeros(105)])
    xo, istop_o, iit_o, r1o, r2o, cost_o = o.cgls(mv, rmv, yo, x0o, niter=10, tol=0.0)
    assert iit == iit_o == 10 and istop == istop_o
    np.testing.assert_allclose(host(xinv.asarray()), xo.asarray(), rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(cost, cost_o, rtol=1e-6, atol=1e-12)
    np.testing.assert_allclose([r1, r2], [r1o, r2o], rtol=1e-6, atol=1e-12)


@pytest.mark.parametrize("dims,h", [(600, 1.0), ((100, 151), 1.0), ((101, 51, 10), 0.4), ((79, 11, 5), 0.4)])
@pytest.mark.parametrize("kind,order", [("forward", 3), ("backward", 3), ("centered", 3), ("centered", 5)])
@pytest.mark.parametrize("edge", [False, True])
@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
@pytest.mark.parametrize("part", ["SCATTER", "BROADCAST"])
def test_first_derivative_operator_grid(pm, dims, h, kind, order, edge, dtype, part):
    # tests/test_derivative.py:33-160, 198-295
    dimsT = (dims,) if np.isscalar(dims) else dims
    n = int(np.prod(dimsT))
    rng = np.random.default_rng(42)
    x = rng.normal(0, 10, n).astype(dtype)
    if np.issubdtype(dtype, np.complexfloating):
        x = x + 1j * rng.normal(0, 10, n)
    Fop = pm.MPIFirstDerivative(dims, sampling=h, kind=kind, edge=edge, order=order, dtype=dtype)
    xd = pm.DistributedArray.to_dist(x, partition=getattr(pm.Partition, part))
    D = o.first_derivative_dense(dimsT[0], h, kind, edge, order)
    X = x.reshape(dimsT[0], -1)
    y = Fop @ xd
    ya = Fop.H @ xd
    assert y.partition is pm.Partition.SCATTER
    np.testing.assert_allclose(host(y.asarray()), (D @ X).ravel(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(host(ya.asarray()), (D.T @ X).ravel(), rtol=1e-12, atol=1e-12)
    u = pm.DistributedArray.to_dist(rng.normal(0, 10, n).astype(dtype))
    v = pm.DistributedArray.to_dist(rng.normal(0, 10, n).astype(dtype))
    assert pm.dottest(Fop, u, v)


def test_first_derivative_errors(pm):
    with pytest.raises(NotImplementedError):
        pm.MPIFirstDerivative(10, kind="sideways")
    with pytest.raises(NotImplementedError):
        pm.MPIFirstDerivative(10, kind="centered", order=7)
    Fop = pm.MPIFirstDerivative(10)
    with pytest.raises(ValueError, match="dimension mismatch"):
        Fop.matvec(pm.DistributedArray.to_dist(np.zeros(11)))
    with pytest.raises(ValueError):
        Fop.matvec(pm.DistributedArray.to_dist(np.zeros(10), partition=pm.Partition.UNSAFE_BROADCAST))


# ---- BlockDiag / VStack / HStack KATs (test_blockdiag.py:24-71, test_stack.py:29-79) ------------
@pytest.mark.parametrize("ny,nx", [(101, 101), (301, 101)])
@pytest.mark.parametrize("dtype", [np.float64, np.complex128, np.float32])
def test_blockdiag_vstack_kats(pm, ny, nx, dtype):
    rank = 0
    A = ((rank + 1) * np.ones((ny, nx))).astype(dtype)
    Op = pm.MatrixMult(A, dtype=dtype)
    BD = pm.MPIBlockDiag([Op])
    assert BD.shape == (ny, nx)
    x = pm.DistributedArray.to_dist(np.ones(nx, dtype=dtype))
    y = BD @ x
    np.testing.assert_allclose(host(y.asarray()), nx * np.ones(ny), rtol=1e-6)
    xa = BD.H @ pm.DistributedArray.to_dist(np.ones(ny, dtype=dtype))
    np.testing.assert_allclose(host(xa.asarray()), ny * np.ones(nx), rtol=1e-6)
    assert pm.dottest(BD, x, pm.DistributedArray.to_dist(np.ones(ny, dtype=dtype)))
    # two blocks on one rank, random data, vs oracle
    rng = np.random.default_rng(1)
    A2 = rng.standard_normal((ny // 2, nx)).astype(dtype)
    BD2 = pm.MPIBlockDiag([Op, pm.MatrixMult(A2)])
    xv = rng.standard_normal(2 * nx).astype(dtype)
    ref = o.blockdiag([[A, A2]], [xv])[0]
    np.testing.assert_allclose(host((BD2 @ pm.DistributedArray.to_dist(xv)).asarray()), ref, rtol=1e-4 if dtype == np.float32 else 1e-12)
    VS = pm.MPIVStack([Op, pm.MatrixMult(A2)])
    xb = pm.DistributedArray.to_dist(rng.standard_normal(nx).astype(dtype), partition=pm.Partition.BROADCAST)
    yv = VS @ xb
    assert yv.partition is pm.Partition.SCATTER
    tol = 1e-4 if dtype == np.float32 else 1e-12
    np.testing.assert_allclose(host(yv.asarray()), o.vstack_matvec([[A, A2]], host(xb.local_array))[0], rtol=tol, atol=tol)
    xr = VS.H @ yv
    assert xr.partition is pm.Partition.BROADCAST
    np.testing.assert_allclose(host(xr.asarray()), o.vstack_rmatvec([[A, A2]], [host(yv.asarray())]), rtol=tol * 10, atol=tol * 100)
    with pytest.raises(ValueError):
        VS @ pm.DistributedArray.to_dist(np.ones(nx, dtype=dtype))
    HS = pm.MPIHStack([pm.MatrixMult(A.T.copy())])
    np.testing.assert_allclose(host((HS @ pm.DistributedArray.to_dist(np.ones(ny, dtype=dtype))).asarray()),
                               ny * np.ones(nx), rtol=1e-6)


# ---- MPIMatrixMult KATs (test_matrixmult.py:37-60, 82-166, 199-271) ----------------------------
@pytest.mark.parametrize("N,K,M,dtype", [(64, 64, 64, np.float64), (37, 37, 37, np.float64), (50, 30, 40, np.float64),
                                         (22, 20, 16, np.complex128), (3, 4, 5, np.float32), (1, 2, 1, np.float64),
                                         (2, 1, 3, np.float32), (64, 48, 1, np.float64)])
@pytest.mark.parametrize("kind", ["summa", "block"])
def test_matrixmult_kats(pm, N, K, M, dtype, kind):
    A = np.arange(N * K, dtype=dtype).reshape(N, K)
    X = np.arange(K * M, dtype=dtype).reshape(K, M)
    if np.issubdtype(dtype, np.complexfloating):
        A = A + 0.5j * A
        X = X + 0.7j * X
    Aop = pm.MPIMatrixMult(A, M, kind=kind, dtype=dtype)
    x = pm.DistributedArray.to_dist(X.ravel())
    y = Aop @ x
    rtol = np.finfo(dtype).resolution * 10
    Yref = (A.astype(np.complex128) @ X.astype(np.complex128)) if np.iscomplexobj(A) else A.astype(np.float64) @ X
    np.testing.assert_allclose(host(y.asarray()).reshape(N, M), Yref, rtol=rtol)
    xadj = Aop.H @ y
    np.testing.assert_allclose(host(xadj.asarray()).reshape(K, M), A.conj().T @ Yref, rtol=rtol * 10)
    with pytest.raises(ValueError):
        Aop @ pm.DistributedArray.to_dist(X.ravel(), partition=pm.Partition.BROADCAST)
    if kind == "summa":
        Rop = pm.MPIMatrixMult(A, M, kind=kind, dtype=dtype, replicate=True)
        np.testing.assert_allclose(host((Rop @ x).asarray()).reshape(N, M), Yref, rtol=rtol)
        np.testing.assert_allclose(host((Rop.H @ y).asarray()).reshape(K, M), A.conj().T @ Yref, rtol=rtol * 10)


# ---- MPIFredholm1 KATs (test_fredholm.py:36-95, 114-167) ---------------------------------------
@pytest.mark.parametrize("nz", [5, 1])
@pytest.mark.parametrize("dtype", [np.float32, np.complex64, np.float64])
@pytest.mark.parametrize("saveGt,usematmul", [(True, True), (False, False)])
def test_fredholm1_kat(pm, nz, dtype, saveGt, usematmul):
    cx = np.issubdtype(dtype, np.complexfloating)
    nsl, nx, ny = 21, 4, 6
    G = np.arange(nsl * nx * ny, dtype=np.float64).reshape(nsl, nx, ny)
    G = (G - 1j * G) if cx else G
    x = (np.ones((nsl, ny, nz)) + (1j if cx else 0)).astype(dtype)
    Fop = pm.MPIFredholm1(G.astype(dtype), nz=nz, saveGt=saveGt, usematmul=usematmul, dtype=dtype)
    xd = pm.DistributedArray.to_dist(x.ravel(), partition=pm.Partition.BROADCAST)
    y = Fop @ xd
    assert y.partition is pm.Partition.BROADCAST
    ref = o.fredholm1([G], x.ravel().astype(G.dtype), nz)
    np.testing.assert_allclose(host(y.asarray()), ref, rtol=1e-5)
    xa = Fop.H @ y
    refa = o.fredholm1([G], ref, nz, adjoint=True)
    np.testing.assert_allclose(host(xa.asarray()), refa, rtol=1e-4)
    with pytest.raises(ValueError):
        Fop @ pm.DistributedArray.to_dist(x.ravel())
    yv = pm.DistributedArray.to_dist(np.ones(nsl * nx * nz, dtype=dtype), partition=pm.Partition.BROADCAST)
    assert pm.dottest(Fop, xd, yv, rtol=1e-4)


# ---- operator algebra (test_linearop.py) ---------------------------------------------------------
def test_operator_algebra(pm):
    rng = np.random.default_rng(0)
    n = 64
    A = rng.standard_normal((n, n)) + 1j * rng.standard_normal((n, n))
    Op = pm.MPIBlockDiag([pm.MatrixMult(A)])
    x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    xd = pm.DistributedArray.to_dist(x)
    chk = lambda got, ref: np.testing.assert_allclose(host(got.asarray()), ref, rtol=1e-11)  # noqa: E731
    chk(Op.H @ xd, A.conj().T @ x)
    chk(Op.T @ xd, A.T @ x)
    chk(Op.conj() @ xd, A.conj() @ x)
    chk((Op * Op) @ xd, A @ (A @ x))
    chk((Op + Op) @ xd, 2 * A @ x)
    chk((Op - Op.H) @ xd, (A - A.conj().T) @ x)
    chk((3j * Op) @ xd, 3j * (A @ x))
    chk((3j * Op).H @ xd, np.conj(3j) * (A.conj().T @ x))
    chk((-Op) @ xd, -(A @ x))
    chk((Op ** 3) @ xd, A @ (A @ (A @ x)))
    chk(pm.asmpilinearoperator(Op) * xd, A @ x)
    with pytest.raises(ValueError):
        Op @ 3.0


# ---- CGLS on BlockDiag (test_solver.py:44-100, 150-196) -----------------------------------------
@pytest.mark.parametrize("ny,nx", [(11, 11), (31, 11)])
@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
def test_cgls_blockdiag_vs_oracle(pm, ny, nx, dtype):
    rng = np.random.default_rng(42)
    A = np.ones((ny, nx), dtype=dtype)
    blk = A.conj().T @ A + 1e-5 * np.eye(nx, dtype=dtype)
    Op = pm.MPIBlockDiag([pm.MatrixMult(blk)])
    xt = rng.normal(1, 10, nx).astype(dtype)
    if np.issubdtype(dtype, np.complexfloating):
        xt = xt + 1j * rng.normal(10, 10, nx)
    y = Op @ pm.DistributedArray.to_dist(xt)
    for x0v in (np.zeros(nx, dtype=dtype), rng.normal(0, 10, nx).astype(dtype)):
        xinv, istop, iit, r1, r2, cost = pm.cgls(Op, y, x0=pm.DistributedArray.to_dist(x0v), niter=nx, tol=1e-5)
        mv = lambda a: o.SimArray(o.blockdiag([[blk]], a.locs))                  # noqa: E731
        rmv = lambda a: o.SimArray(o.blockdiag([[blk]], a.locs, adjoint=True))   # noqa: E731
        xo, istop_o, iit_o, r1o, r2o, cost_o = o.cgls(mv, rmv, mv(o.SimArray([xt])), o.SimArray([x0v]), niter=nx, tol=1e-5)
        assert (istop, iit) == (istop_o, iit_o)
        np.testing.assert_allclose(host(xinv.asarray()), xo.asarray(), rtol=1e-6, atol=1e-8)
        np.testing.assert_allclose(cost, cost_o, rtol=1e-5, atol=1e-8)
    xcg, itcg, costcg = pm.cg(Op, y, x0=pm.DistributedArray.to_dist(np.zeros(nx, dtype=dtype)), niter=nx, tol=1e-5)
    xo, ito, costo = o.cg(mv, mv(o.SimArray([xt])), o.SimArray([np.zeros(nx, dtype=dtype)]), niter=nx, tol=1e-5)
    assert itcg == ito
    np.testing.assert_allclose(host(xcg.asarray()), xo.asarray(), rtol=1e-6, atol=1e-8)


def test_cgls_config3_single_block_fp32(pm):
    """BASELINE config 3 restricted to one 4096x4096 float32 block: 50 iterations reach the
    float64 oracle solution to 1e-6 relative"""
    n = 4096
    A = (np.random.default_rng(100).standard_normal((n, n), dtype=np.float32) / 128 + 2 * np.eye(n, dtype=np.float32))
    xt = np.random.default_rng(7).standard_normal(n).astype(np.float32)
    Op = pm.MPIBlockDiag([pm.MatrixMult(A)])
    y = Op @ pm.DistributedArray.to_dist(xt)
    xinv, istop, iit, r1, r2, cost = pm.cgls(Op, y, x0=pm.DistributedArray.to_dist(np.zeros(n, np.float32)), niter=50, tol=0.0)
    assert iit == 50
    A64 = A.astype(np.float64)
    mv = lambda a: o.SimArray([A64 @ a.locs[0]])       # noqa: E731
    rmv = lambda a: o.SimArray([A64.T @ a.locs[0]])    # noqa: E731
    xo, *_rest, cost_o = o.cgls(mv, rmv, o.SimArray([A64 @ xt.astype(np.float64)]), o.SimArray([np.zeros(n)]), niter=50, tol=0.0)
    rel = np.linalg.norm(host(xinv.asarray()) - xo.asarray()) / np.linalg.norm(xo.asarray())
    assert rel < 1e-5, rel
    assert np.linalg.norm(host(xinv.asarray()) - xt) / np.linalg.norm(xt) < 1e-5


def test_cgls_graph_capture_survives_solver_turnover(pm):
    """every solver captures its iteration into the process-wide graph pool: a capture must still succeed after the
    previous solver (and its graph) has been freed (regression: torch asserts 'use_count > 0' when a capture joins a
    pool no live graph references), and torch's RNG must stay usable afterwards"""
    import gc
    from pylops_mpi_b200.optimization.cls_basic import CGLS
    n = 256
    A = (np.random.default_rng(3).standard_normal((n, n)) / 64 + 2 * np.eye(n)).astype(np.float32)
    xt = np.random.default_rng(4).standard_normal(n).astype(np.float32)
    Op = pm.MPIBlockDiag([pm.MatrixMult(A)])
    y = Op @ pm.DistributedArray.to_dist(xt)
    for _ in range(3):
        solver = CGLS(Op)
        x = solver.setup(y=y, x0=pm.DistributedArray.to_dist(np.zeros(n, np.float32)), niter=20, damp=0.0, tol=0.0)
        x = solver.run(x, 20)
        solver.finalize()
        assert solver.graph_error is None, solver.graph_error
        assert solver.graph_replays >= 18
        assert np.linalg.norm(host(x.asarray()) - xt) / np.linalg.norm(xt) < 1e-2
        del solver, x
        gc.collect()
        torch.randn(8, device="cuda")          # RNG not left in capture mode


# ---- MPIMatrixMult bf16 -> fp32 (BASELINE config 4, reduced size) --------------------------------
@pytest.mark.parametrize("kind", ["summa", "block"])
@pytest.mark.parametrize("M", [1, 256])
def test_matrixmult_bf16(pm, kind, M):
    N = K = 1024
    A = (np.random.default_rng(1).standard_normal((N, K)) / 181).astype(np.float32)
    At = torch.as_tensor(A).to(torch.bfloat16)
    X = np.random.default_rng(2).standard_normal((K, M)).astype(np.float32)
    Xb = torch.as_tensor(X).to(torch.bfloat16).float().numpy() if M > 1 else X
    Aop = pm.MPIMatrixMult(At, M, kind=kind, dtype="bfloat16")
    x = pm.DistributedArray.to_dist(X.ravel())
    y = Aop @ x
    A64 = At.double().numpy()
    ref = A64 @ Xb.astype(np.float64)
    scale = np.abs(A64) @ np.abs(Xb.astype(np.float64))
    err = np.abs(host(y.asarray()).reshape(N, M) - ref)
    assert np.all(err <= scale * K * 6e-8 + 1e-6)
    ya = Aop.H @ y
    yb = torch.as_tensor(host(y.asarray()).reshape(N, M)).to(torch.bfloat16).double().numpy() if M > 1 else host(y.asarray()).reshape(N, M).astype(np.float64)
    refa = A64.T @ yb
    erra = np.abs(host(ya.asarray()).reshape(K, M) - refa)
    assert np.all(erra <= (np.abs(A64.T) @ np.abs(yb)) * N * 6e-8 + 1e-6)


# ---- MPIMDC ("next" row f1; reference-chain fixtures are in test_golden.py; here: oracle + adjointness) ------
@pytest.mark.parametrize("twosided", [True, False])
@pytest.mark.parametrize("dtype", [np.complex64, np.complex128])
def test_mdc_pipeline(pm, twosided, dtype):
    rng = np.random.default_rng(11)
    ns, nr, nv, nt = 6, 5, 3, 31 if twosided else 32
    nfft = int(np.ceil((nt + 1) / 2))
    nfmax = nfft - 3
    G = (rng.standard_normal((nfmax, ns, nr)) + 1j * rng.standard_normal((nfmax, ns, nr))).astype(dtype)
    rdt = np.float32 if dtype == np.complex64 else np.float64
    Mop = pm.MPIMDC(G, nt=nt, nv=nv, nfreq=nfmax, dt=0.004, dr=2.0, twosided=twosided)
    assert Mop.shape == (nt * ns * nv, nt * nr * nv)
    m = rng.standard_normal(nt * nr * nv).astype(rdt)
    md = pm.DistributedArray.to_dist(m, partition=pm.Partition.BROADCAST)
    d = Mop @ md
    assert d.partition is pm.Partition.BROADCAST
    ref = o.mdc([G.astype(np.complex128)], m.astype(np.float64), nt, nv, twosided, False, dt=0.004, dr=2.0)
    tol = 2e-4 if dtype == np.complex64 else 1e-11
    np.testing.assert_allclose(host(d.asarray()).real, ref, rtol=tol, atol=tol * np.abs(ref).max())
    dd = rng.standard_normal(nt * ns * nv).astype(rdt)
    ma = Mop.H @ pm.DistributedArray.to_dist(dd, partition=pm.Partition.BROADCAST)
    refa = o.mdc([G.astype(np.complex128)], dd.astype(np.float64), nt, nv, twosided, True, dt=0.004, dr=2.0)
    np.testing.assert_allclose(host(ma.asarray()).real, refa, rtol=tol, atol=tol * np.abs(refa).max())
    # adjointness of the whole chain on real vectors
    lhs = float(np.dot(host(d.asarray()).real.astype(np.float64), dd.astype(np.float64)))
    rhs = float(np.dot(m.astype(np.float64), host(ma.asarray()).real.astype(np.float64)))
    assert abs(lhs - rhs) <= (1e-3 if dtype == np.complex64 else 1e-10) * max(abs(lhs), abs(rhs), 1.0)
    with pytest.raises(ValueError):
        pm.MPIMDC(G, nt=30, nv=nv, nfreq=nfmax, twosided=True)


# ---- MPIGradient / stacked glue ("next" row f3, minimal) --------------------------------------------------
@pytest.mark.parametrize("dims", [(20, 17), (12, 9, 10)])
@pytest.mark.parametrize("kind,edge", [("centered", True), ("forward", False)])
def test_gradient_stacked(pm, dims, kind, edge):
    rng = np.random.default_rng(2)
    n = int(np.prod(dims))
    x = rng.standard_normal(n)
    samp = tuple(1.0 + 0.5 * i for i in range(len(dims)))
    Gop = pm.MPIGradient(dims, sampling=samp, edge=edge, kind=kind, dtype=np.float64)
    y = Gop.matvec(pm.DistributedArray.to_dist(x))
    assert isinstance(y, pm.StackedDistributedArray) and y.narrays == len(dims)
    X = x.reshape(dims)
    refs = [o.derivative_along_axis(X, ax, o.first_derivative_dense(dims[ax], samp[ax], kind, edge, 3)).ravel()
            for ax in range(len(dims))]
    for ax in range(len(dims)):
        np.testing.assert_allclose(host(y[ax].asarray()), refs[ax], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(host(y.asarray()), np.concatenate(refs), rtol=1e-12, atol=1e-12)
    xa = Gop.rmatvec(y)
    refa = sum(o.derivative_along_axis(refs[ax].reshape(dims), ax, o.first_derivative_dense(dims[ax], samp[ax], kind, edge, 3).T)
               for ax in range(len(dims)))
    np.testing.assert_allclose(host(xa.asarray()), refa.ravel(), rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(y.dot(y)[0], sum(np.dot(r, r) for r in refs), rtol=1e-12)
    np.testing.assert_allclose(y.norm()[0], np.sqrt(sum(np.dot(r, r) for r in refs)), rtol=1e-12)
    z = y + y * 2.0 - y
    np.testing.assert_allclose(host(z.asarray()), 2 * np.concatenate(refs), rtol=1e-12, atol=1e-12)


def test_stacked_operator_algebra(pm):
    """MPIStackedBlockDiag / MPIStackedVStack and the MPIStackedLinearOperator algebra
    (StackedLinearOperator.py:117-228, test_stackedlinearop.py) against dense NumPy"""
    rng = np.random.default_rng(11)
    n1, n2 = 12, 9
    A1, A2 = rng.standard_normal((n1, n1)), rng.standard_normal((n2, n2))
    B1, B2 = rng.standard_normal((7, n1)), rng.standard_normal((5, n1))
    mk = lambda A: pm.MPIBlockDiag([pm.MatrixMult(A)])                      # noqa: E731
    SB = pm.MPIStackedBlockDiag([mk(A1), mk(A2)])
    SV = pm.MPIStackedVStack([mk(B1), mk(B2)])
    assert SB.shape == (n1 + n2, n1 + n2) and SV.shape == (12, n1)
    x1, x2 = rng.standard_normal(n1), rng.standard_normal(n2)
    xs = pm.StackedDistributedArray([pm.DistributedArray.to_dist(x1), pm.DistributedArray.to_dist(x2)])
    Dm = np.block([[A1, np.zeros((n1, n2))], [np.zeros((n2, n1)), A2]])
    xf = np.concatenate([x1, x2])
    tol = dict(rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(host((SB @ xs).asarray()), Dm @ xf, **tol)
    np.testing.assert_allclose(host((SB.H @ xs).asarray()), Dm.T @ xf, **tol)
    np.testing.assert_allclose(host((SB.T @ xs).asarray()), Dm.T @ xf, **tol)
    np.testing.assert_allclose(host((SB.conj() @ xs).asarray()), Dm @ xf, **tol)
    np.testing.assert_allclose(host(((2.5 * SB) @ xs).asarray()), 2.5 * Dm @ xf, **tol)
    np.testing.assert_allclose(host(((-SB) @ xs).asarray()), -Dm @ xf, **tol)
    np.testing.assert_allclose(host(((SB + SB) @ xs).asarray()), 2 * Dm @ xf, **tol)
    np.testing.assert_allclose(host(((SB - 0.5 * SB) @ xs).asarray()), 0.5 * Dm @ xf, **tol)
    np.testing.assert_allclose(host(((SB ** 3) @ xs).asarray()), Dm @ Dm @ Dm @ xf, rtol=1e-10, atol=1e-9)
    np.testing.assert_allclose(host(((SB * SB).H @ xs).asarray()), (Dm @ Dm).T @ xf, rtol=1e-10, atol=1e-9)
    # VStack: model is a plain DistributedArray, data is stacked; product with a BlockDiag on the data side
    Vm = np.vstack([B1, B2])
    xd = pm.DistributedArray.to_dist(x1)
    yv = SV @ xd
    np.testing.assert_allclose(host(yv.asarray()), Vm @ x1, **tol)
    np.testing.assert_allclose(host((SV.H @ yv).asarray()), Vm.T @ (Vm @ x1), rtol=1e-10, atol=1e-9)
    np.testing.assert_allclose(host(((SV.H * SV) @ xd).asarray()), Vm.T @ Vm @ x1, rtol=1e-10, atol=1e-9)
    with pytest.raises(ValueError, match="dimension mismatch"):
        SB.matvec(xd)
    with pytest.raises(ValueError, match="both operands cannot be MPIStackedVStack"):
        SV * SV
    with pytest.raises(ValueError, match="Scalar not allowed"):
        SB @ 2.0
    # sparsity solver on a stacked operator (generic, unfused path with stacked model/data)
    eig = pm.power_iteration(SB.H * SB, niter=400, tol=1e-13, dtype=np.float64, b_k=xs.empty_like())[0]
    np.testing.assert_allclose(np.abs(eig), np.linalg.norm(Dm, 2) ** 2, rtol=1e-3)
    y = SB @ xs
    x0 = pm.StackedDistributedArray([pm.DistributedArray.to_dist(np.zeros(n1)), pm.DistributedArray.to_dist(np.zeros(n2))])
    alpha = 1.0 / np.linalg.norm(Dm, 2) ** 2
    xi, it, cost = pm.ista(SB, y, x0, niter=25, eps=0.1, alpha=alpha, tol=1e-12)
    xo, ito, co = o.ista(Dm, Dm @ xf, np.zeros(n1 + n2), 25, 0.1, alpha, 1e-12, "soft")
    assert it == ito
    np.testing.assert_allclose(cost, co, rtol=1e-9)
    np.testing.assert_allclose(host(xi.asarray()), xo, rtol=1e-9, atol=1e-9)


# ---- round 2: mixed dtypes (ADVICE high), operators on promoted data, stacked CG / CGLS, tensor-core Fredholm -------
def test_mixed_dtype_arithmetic_matches_the_reference_casting(pm):
    """float64 +/- float32, real * complex, dot with mixed dtypes.  The reference computes ``self.local_array (op)
    other.local_array`` (NumPy promotion) and ASSIGNS it into an array of ``self.dtype`` (DistributedArray.py:603-652):
    the result has the LEFT operand's dtype, complex into real keeps the real part with a ComplexWarning.  Never a
    reinterpreted buffer (round-1 ADVICE)."""
    import warnings
    rng = np.random.default_rng(3)
    a64, b32 = rng.standard_normal(1001), rng.standard_normal(1001).astype(np.float32)
    c128 = (rng.standard_normal(1001) + 1j * rng.standard_normal(1001))
    A, B, Cc = (pm.DistributedArray.to_dist(v) for v in (a64, b32, c128))

    def ref(left, expr):
        out = np.empty_like(left)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out[:] = expr
        return out
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", np.exceptions.ComplexWarning)
        cases = [((A - B), ref(a64, a64 - b32)), ((B + A), ref(b32, b32 + a64)), ((A * B), ref(a64, a64 * b32)),
                 ((B * Cc), ref(b32, b32 * c128)), ((A + Cc), ref(a64, a64 + c128)), ((Cc - A), ref(c128, c128 - a64)),
                 ((A * (1 + 2j)), ref(a64, a64 * (1 + 2j)))]
    for got, want in cases:
        assert got.dtype == want.dtype, (got.dtype, want.dtype)
        np.testing.assert_allclose(host(got.asarray()), want, rtol=1e-6 if want.dtype == np.float32 else 1e-12)
    np.testing.assert_allclose(A.dot(B)[0], np.dot(a64, b32), rtol=1e-12)
    A2 = A.copy()
    A2 += B
    assert A2.dtype == np.float64
    np.testing.assert_allclose(host(A2.asarray()), a64 + b32, rtol=1e-12)
    B2 = B.copy()
    B2 -= A
    assert B2.dtype == np.float32
    np.testing.assert_allclose(host(B2.asarray()), (b32 - a64).astype(np.float32), rtol=1e-6)
    with pytest.warns(np.exceptions.ComplexWarning):
        A2 += Cc                                     # self[:] = self + other: real part kept, warning
    np.testing.assert_allclose(host(A2.asarray()), a64 + b32 + c128.real, rtol=1e-12)


def test_cg_with_float64_x0_and_float32_operator(pm):
    """the ADVICE example: default float64 x0 with a float32 operator must not mix buffers in axpy_/xpby_"""
    n = 64
    A = np.random.default_rng(5).standard_normal((n, n)).astype(np.float32)
    A = A @ A.T / n + 2 * np.eye(n, dtype=np.float32)
    Op = pm.MPIBlockDiag([pm.MatrixMult(A)])
    xt = np.random.default_rng(6).standard_normal(n)
    y = Op @ pm.DistributedArray.to_dist(xt.astype(np.float32))
    x0 = pm.DistributedArray.to_dist(np.zeros(n))   # float64
    xinv, iit, cost = pm.cg(Op, y, x0=x0, niter=12, tol=0.0)
    np.testing.assert_allclose(host(xinv.asarray()), xt, rtol=0, atol=1e-4 * np.abs(xt).max())
    xinv2, *_ = pm.cgls(Op, y, x0=x0, niter=25, tol=0.0)
    np.testing.assert_allclose(host(xinv2.asarray()), xt, rtol=0, atol=1e-3 * np.abs(xt).max())


def test_real_block_applied_to_complex_data_keeps_imaginary_part(pm):
    """result_type(op, x): a real MatrixMult block inside a complex-typed MPIBlockDiag (ADVICE medium)"""
    rng = np.random.default_rng(8)
    A = rng.standard_normal((31, 17))
    xc = rng.standard_normal(17) + 1j * rng.standard_normal(17)
    Op = pm.MPIBlockDiag([pm.MatrixMult(A)], dtype=np.complex128)
    y = Op @ pm.DistributedArray.to_dist(xc)
    np.testing.assert_allclose(host(y.asarray()), A @ xc, rtol=1e-12)
    ya = Op.H @ y
    np.testing.assert_allclose(host(ya.asarray()), A.T @ (A @ xc), rtol=1e-12)
    # mixed float32 / float64 blocks in one BlockDiag: output dtype = result_type of the blocks
    B32 = rng.standard_normal((9, 5)).astype(np.float32)
    Op2 = pm.MPIBlockDiag([pm.MatrixMult(A), pm.MatrixMult(B32)])
    xv = rng.standard_normal(22)
    y2 = Op2 @ pm.DistributedArray.to_dist(xv)
    assert y2.dtype == np.float64
    np.testing.assert_allclose(host(y2.asarray()), np.concatenate([A @ xv[:17], B32.astype(np.float64) @ xv[17:]]),
                               rtol=1e-5, atol=1e-5)          # the float32 block runs a float32 GEMV


def test_local_operator_typeerror_is_not_swallowed(pm):
    """a TypeError raised INSIDE an operator must propagate (out= support is detected by type, not by catching)"""
    class Bad(pm.local.LocalOperator):
        shape = (4, 4)
        dtype = np.float64

        def matvec(self, x, out=None):
            raise TypeError("genuine bug inside the operator")
    with pytest.raises(TypeError, match="genuine bug"):
        pm.MPIBlockDiag([Bad()]) @ pm.DistributedArray.to_dist(np.ones(4))


def test_cg_cgls_on_stacked_arrays(pm):
    """reference tests/test_solver.py:303-427: CG / CGLS with StackedDistributedArray models (MPIStackedBlockDiag)"""
    rng = np.random.default_rng(11)
    n1, n2 = 13, 7
    A1 = rng.standard_normal((n1, n1)); A1 = A1 @ A1.T + n1 * np.eye(n1)
    A2 = rng.standard_normal((n2, n2)); A2 = A2 @ A2.T + n2 * np.eye(n2)
    Op = pm.MPIStackedBlockDiag([pm.MPIBlockDiag([pm.MatrixMult(A1)]), pm.MPIBlockDiag([pm.MatrixMult(A2)])])
    x1, x2 = rng.standard_normal(n1), rng.standard_normal(n2)
    xs = pm.StackedDistributedArray([pm.DistributedArray.to_dist(x1), pm.DistributedArray.to_dist(x2)])
    y = Op.matvec(xs)
    x0 = pm.StackedDistributedArray([pm.DistributedArray.to_dist(np.zeros(n1)), pm.DistributedArray.to_dist(np.zeros(n2))])
    xcg, iit, cost = pm.cg(Op, y, x0=x0, niter=30, tol=0.0)
    np.testing.assert_allclose(host(xcg.asarray()), np.concatenate([x1, x2]), rtol=1e-8, atol=1e-10)
    xls, istop, iit, r1, r2, cost = pm.cgls(Op, y, x0=x0, niter=60, tol=0.0)
    np.testing.assert_allclose(host(xls.asarray()), np.concatenate([x1, x2]), rtol=1e-6, atol=1e-8)
    # same numbers as the oracle's CGLS on the dense block-diagonal system (the reference's own recurrences)
    import scipy.linalg
    Ad = scipy.linalg.block_diag(A1, A2)
    mv = lambda a: o.SimArray([Ad @ a.locs[0]])       # noqa: E731
    rmv = lambda a: o.SimArray([Ad.T @ a.locs[0]])    # noqa: E731
    xo, *_r, cost_o = o.cgls(mv, rmv, o.SimArray([Ad @ np.concatenate([x1, x2])]), o.SimArray([np.zeros(n1 + n2)]), niter=10, tol=0.0)
    xl10, *_r2, cost10 = pm.cgls(Op, y, x0=x0, niter=10, tol=0.0)
    np.testing.assert_allclose(cost10, cost_o, rtol=1e-8)
    np.testing.assert_allclose(host(xl10.asarray()), xo.asarray(), rtol=1e-8, atol=1e-10)


@pytest.mark.parametrize("shape", [(21, 4, 6, 5), (5, 100, 70, 9), (2, 129, 257, 65), (3, 128, 128, 64)])
@pytest.mark.parametrize("dtype", [np.complex64, np.float32])
def test_fredholm1_tensor_core_path(pm, monkeypatch, shape, dtype):
    """MPIFredholm1 on the tensor cores (csrc/fredholm_tc.cu; TC_MIN_PRODUCTS = 0 puts every shape there) vs the oracle
    in complex128 / float64: 1e-5 of the largest entry per output column (north_star tolerance for complex64)"""
    monkeypatch.setattr(pm.signalprocessing.Fredholm1, "TC_MIN_PRODUCTS", 0)
    nsl, nx, ny, nz = shape
    rng = np.random.default_rng(13)
    G = rng.standard_normal((nsl, nx, ny))
    x = rng.standard_normal((nsl, ny, nz))
    if dtype is np.complex64:
        G = G + 1j * rng.standard_normal((nsl, nx, ny))
        x = x + 1j * rng.standard_normal((nsl, ny, nz))
    G, x = G.astype(dtype), x.astype(dtype)
    Fr = pm.MPIFredholm1(G, nz=nz, dtype=dtype)
    assert Fr._plan is not None
    xd = pm.DistributedArray.to_dist(x.ravel(), partition=pm.Partition.BROADCAST)
    wide = np.complex128 if dtype is np.complex64 else np.float64
    refy = o.fredholm1([G.astype(wide)], x.ravel().astype(wide), nz)
    y = Fr @ xd
    got = host(y.local_array).reshape(nsl, nx, nz)
    ref = refy.reshape(nsl, nx, nz)
    assert np.all(np.abs(got - ref).max(axis=1) <= 1e-5 * np.abs(ref).max(axis=1))
    refx = o.fredholm1([G.astype(wide)], refy, nz, adjoint=True).reshape(nsl, ny, nz)
    gotx = host((Fr.H @ y).local_array).reshape(nsl, ny, nz)
    assert np.all(np.abs(gotx - refx).max(axis=1) <= 2e-5 * np.abs(refx).max(axis=1))
    assert pm.dottest(Fr, pm.DistributedArray.to_dist(x.ravel(), partition=pm.Partition.BROADCAST),
                      pm.DistributedArray.to_dist(refy.astype(dtype), partition=pm.Partition.BROADCAST), rtol=1e-4)


def test_fredholm1_kat_on_tensor_cores(pm, monkeypatch):
    """tests/test_fredholm.py:36-95 arange KAT through the tensor-core path (exactly representable inputs)"""
    monkeypatch.setattr(pm.signalprocessing.Fredholm1, "TC_MIN_PRODUCTS", 0)
    for nz in (5, 1):
        for dtype in (np.float32, np.complex64):
            cx = dtype is np.complex64
            G = np.arange(21 * 4 * 6, dtype=np.float64).reshape(21, 4, 6)
            G = (G - 1j * G) if cx else G
            xv = (np.ones((21, 6, nz)) + (1j if cx else 0))
            Fr = pm.MPIFredholm1(G.astype(dtype), nz=nz, dtype=dtype)
            y = Fr @ pm.DistributedArray.to_dist(xv.ravel().astype(dtype), partition=pm.Partition.BROADCAST)
            refy = o.fredholm1([G], xv.ravel().astype(G.dtype), nz)
            np.testing.assert_allclose(host(y.local_array), refy, rtol=1e-5)
            np.testing.assert_allclose(host((Fr.H @ y).local_array), o.fredholm1([G], refy, nz, adjoint=True), rtol=1e-4)


def test_fredholm1_baseline_size_complex64_vs_complex128(pm):
    """SURVEY 8(d) C5 at full per-GPU size: 64 slices of 256 x 256 x 64 complex64 vs complex128, 1e-5 of max"""
    nsl, ns, nr, nv = 64, 256, 256, 64
    g = torch.Generator(device="cuda").manual_seed(3)
    G = torch.randn(nsl, ns, nr, device="cuda", dtype=torch.complex64, generator=g)
    xm = torch.randn(nsl * nr * nv, device="cuda", dtype=torch.complex64, generator=g)
    Fr = pm.MPIFredholm1(G, nz=nv, dtype=np.complex64)
    assert Fr._plan is not None          # the tensor-core path is the default at this size
    xd = pm.DistributedArray(global_shape=xm.numel(), partition=pm.Partition.BROADCAST, dtype=np.complex64)
    xd.local_array.copy_(xm)
    y = Fr @ xd
    ref = torch.matmul(G.to(torch.complex128), xm.view(nsl, nr, nv).to(torch.complex128))
    got = y.local_array.view(nsl, ns, nv).to(torch.complex128)
    assert ((got - ref).abs().amax(dim=1) <= 1e-5 * ref.abs().amax(dim=1)).all()
    ya = Fr.H @ y
    refa = torch.matmul(G.to(torch.complex128).conj().transpose(1, 2), got)
    gota = ya.local_array.view(nsl, nr, nv).to(torch.complex128)
    assert ((gota - refa).abs().amax(dim=1) <= 1e-5 * refa.abs().amax(dim=1)).all()


def test_parity_check_set_runs_clean_on_one_rank(pm):
    """the driver-visible parity set of bench.py (tests/parity_checks.py) at world size 1"""
    import parity_checks
    res = parity_checks.run_all(pm, pm.get_comm_world(), full_size=True)
    assert res["failed"] == 0, res["failures"]
    assert res["checked"] >= 10


@pytest.mark.parametrize("twosided", [True, False])
def test_mdc_frequency_domain_variant(pm, twosided):
    """data_domain="frequency" (scattered band-limited spectrum, no Allgather in the forward apply): the remaining
    stages F1^H I1^H applied to its output reproduce the reference-chain MPIMDC / oracle.mdc; adjoint by dot-test;
    CGLS on the spectrum-domain residual gives the time-domain MDD iterates for a physical (real-DC) kernel"""
    rng = np.random.default_rng(17)
    ns, nr, nv, nt = 7, 6, 3, 31 if twosided else 32
    nfft = int(np.ceil((nt + 1) / 2))
    nfmax = nfft - 3
    gt = rng.standard_normal((nt, ns, nr))                                 # real time-domain kernel -> real DC slice
    G = np.fft.rfft(gt, n=nt, axis=0)[:nfmax].astype(np.complex128)
    Mt = pm.MPIMDC(G, nt=nt, nv=nv, nfreq=nfmax, dt=0.004, dr=2.0, twosided=twosided)
    Mf = pm.MPIMDC(G, nt=nt, nv=nv, nfreq=nfmax, dt=0.004, dr=2.0, twosided=twosided, data_domain="frequency")
    m = rng.standard_normal(nt * nr * nv)
    md = pm.DistributedArray.to_dist(m, partition=pm.Partition.BROADCAST)
    dt_ = Mt @ md
    df = Mf @ md
    assert df.partition is pm.Partition.SCATTER and df.global_shape == (nfmax * ns * nv,)
    ref = o.mdc([G], m, nt, nv, twosided, False, dt=0.004, dr=2.0)
    np.testing.assert_allclose(host(dt_.asarray()).real, ref, rtol=1e-10, atol=1e-10 * np.abs(ref).max())
    # the spectrum the frequency-domain operator returns is I1 F1 of the time-domain data (up to the imag DC part)
    spec = host(Mf.data_to_frequency(dt_).asarray())
    got = host(df.asarray())
    sl = slice(ns * nv, None)                                              # all bins but DC
    np.testing.assert_allclose(got[sl], spec[sl], rtol=1e-9, atol=1e-9 * np.abs(spec).max())
    np.testing.assert_allclose(got[:ns * nv].real, spec[:ns * nv].real, rtol=1e-9, atol=1e-9 * np.abs(spec).max())
    # adjoint
    u = pm.DistributedArray.to_dist(rng.standard_normal(nt * nr * nv), partition=pm.Partition.BROADCAST)
    v = Mf @ pm.DistributedArray.to_dist(rng.standard_normal(nt * nr * nv), partition=pm.Partition.BROADCAST)
    lhs = np.vdot(host((Mf @ u).asarray()), host(v.asarray()))
    rhs = np.vdot(host(u.asarray()), host((Mf.H @ v).asarray()))
    assert abs(lhs.real - rhs.real) <= 1e-9 * max(abs(lhs), 1.0)
    # MDD: same iterates from the time-domain and the spectrum-domain residuals
    x0 = pm.DistributedArray.to_dist(np.zeros(nt * nr * nv), partition=pm.Partition.BROADCAST)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", np.exceptions.ComplexWarning)
        xt, istop, iit, r1, r2, cost_t = pm.cgls(Mt, dt_, x0=x0, niter=8, tol=0.0)
        xf, *_ = pm.cgls(Mf, Mf.data_to_frequency(dt_), x0=x0, niter=8, tol=0.0)
    # the reference's CGLS recurrences over the oracle's MDC (real model, complex-typed data: the packed device
    # scalars of the fused solver must keep (re, im) slots apart) -- iterate AND cost history
    mv = lambda a: o.SimArray([o.mdc([G], a.locs[0], nt, nv, twosided, False, dt=0.004, dr=2.0)])    # noqa: E731
    rmv = lambda a: o.SimArray([o.mdc([G], a.locs[0], nt, nv, twosided, True, dt=0.004, dr=2.0)])    # noqa: E731
    xo, *_r, cost_o = o.cgls(mv, rmv, o.SimArray([ref]), o.SimArray([np.zeros(nt * nr * nv)]), niter=8, tol=0.0)
    np.testing.assert_allclose(cost_t, cost_o, rtol=1e-8)
    np.testing.assert_allclose(host(xt.asarray()).real, xo.asarray(), rtol=1e-7, atol=1e-9 * np.abs(xo.asarray()).max())
    np.testing.assert_allclose(host(xf.asarray()).real, host(xt.asarray()).real, rtol=1e-6,
                               atol=1e-6 * np.abs(host(xt.asarray())).max())


@pytest.mark.parametrize("shape,part_axis,norm_axis", [((500, 501), 1, 0), ((500, 501), 1, 1), ((600, 600), 0, 1),
                                                       ((600, 600), 0, 0), ((1200,), 0, 0), ((37, 9, 14), 1, 2),
                                                       ((37, 9, 14), 1, 1), ((64, 300), 0, 1)])
@pytest.mark.parametrize("dtype", [np.float64, np.complex128, np.float32])
def test_axis_norms_on_kernels(pm, shape, part_axis, norm_axis, dtype):
    """tests/test_distributedarray.py:211-222 with axis=...: DistributedArray.norm(ord, axis) through b2_norm_axis"""
    rng = np.random.default_rng(5)
    a = rng.normal(100, 100, shape).astype(dtype)
    if np.issubdtype(dtype, np.complexfloating):
        a = a + 1j * rng.normal(50, 50, shape)
    a.ravel()[::7] = 0
    for partition in (pm.Partition.SCATTER, pm.Partition.BROADCAST):
        A = pm.DistributedArray.to_dist(a, partition=partition, axis=part_axis)
        for ord_ in (1, 2, np.inf, -np.inf, 0, 3):
            got = host(A.norm(ord_, norm_axis))
            ref = np.linalg.norm(a.astype(np.complex128 if np.iscomplexobj(a) else np.float64), ord=ord_, axis=norm_axis)
            np.testing.assert_allclose(got, ref, rtol=1e-5 if dtype == np.float32 else 1e-12)


def test_graft_entry_smoke(pm):
    """the driver's smoke() entry point (config-1 KAT / adjoint / cgls + one BlockDiag block vs the oracle)"""
    import __graft_entry__ as g
    g.smoke()
