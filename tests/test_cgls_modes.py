"""CGLS has one fused iteration (``CGLS._body``) and every way of running it gives the same bits: ``run()`` replaying
it as a CUDA graph, ``run()`` executing it eagerly for an operator that is not graph-safe, a ``step()`` loop,
``show=True`` and a callback (both of which run per iteration)."""
import numpy as np
import pytest
from op_checks import host

pytestmark = pytest.mark.gpu

NITER = 30
FIELDS = ("x", "cost", "cost1", "iiter", "istop", "r1norm", "r2norm")


@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


def problem(pm, dtype, layout):
    """(graph-safe operator, the same operator behind a plain LocalOperator, y, x0) on seeded data; "vstack" has a
    BROADCAST model, whose updates take the unfused update + reduction path"""
    from pylops_mpi_b200.local import LocalOperator

    class Delegate(LocalOperator):
        def __init__(self, op):
            self.op, self.shape, self.dtype = op, op.shape, op.dtype

        def _matvec(self, x):
            return self.op.matvec(x)

        def _rmatvec(self, x):
            return self.op.rmatvec(x)

    rng = np.random.default_rng(21)

    def rand(*shape):
        a = rng.standard_normal(shape)
        return (a + 1j * rng.standard_normal(shape) if dtype == "complex128" else a).astype(dtype)

    blocks = [pm.MatrixMult(rand(80, 64)) for _ in range(2)]
    if layout == "blockdiag":
        Op, Eop = pm.MPIBlockDiag(blocks), pm.MPIBlockDiag([Delegate(b) for b in blocks])
        dist = pm.DistributedArray.to_dist
    else:
        Op, Eop = pm.MPIVStack(blocks), pm.MPIVStack([Delegate(b) for b in blocks])

        def dist(a):
            return pm.DistributedArray.to_dist(a, partition=pm.Partition.BROADCAST)
    y = Op @ dist(rand(Op.shape[1]))
    return Op, Eop, y, dist(rand(Op.shape[1]))


def stop_tol(Op, y, x0, damp, first):
    """a tol whose stopping test fires after iteration T >= first, T not a multiple of the 8-iteration block"""
    from pylops_mpi_b200.optimization.cls_basic import CGLS
    s = CGLS(Op)
    x = s.setup(y=y, x0=x0, niter=NITER, damp=damp, tol=0.0)
    ks = [s.kold]
    for _ in range(NITER - 1):
        x = s.step(x)
        ks.append(s.kold)
    T = next(t for t in range(first, NITER) if t % 8 and ks[t] < min(ks[:t]))
    return (ks[T] + min(ks[:T])) / 2, T


def solve(Op, y, x0, damp, tol, mode):
    from pylops_mpi_b200.optimization.cls_basic import CGLS
    s = CGLS(Op)
    if mode == "callback":
        s.callback = lambda x: None             # what cgls(callback=...) does
    if mode == "step":
        x = s.setup(y=y, x0=x0, niter=NITER, damp=damp, tol=tol)
        while s.iiter < NITER and s.kold > tol:
            x = s.step(x)
        s.finalize()
    else:
        x = s.solve(y, x0, niter=NITER, damp=damp, tol=tol, show=mode == "show")[0]
    return s, {"x": host(x.asarray()), "cost": np.asarray(s.cost), "cost1": np.asarray(s.cost1), "iiter": s.iiter,
               "istop": s.istop, "r1norm": s.r1norm, "r2norm": s.r2norm}


@pytest.mark.parametrize("layout", ["blockdiag", "vstack"])
@pytest.mark.parametrize("stop", [None, 3, 10])
@pytest.mark.parametrize("damp", [0.0, 0.5])
@pytest.mark.parametrize("dtype", ["float32", "float64", "complex128"])
def test_cgls_modes_give_identical_bits(pm, capsys, dtype, damp, stop, layout):
    Op, Eop, y, x0 = problem(pm, dtype, layout)
    tol, T = (0.0, NITER) if stop is None else stop_tol(Op, y, x0, damp, stop)
    s, ref = solve(Op, y, x0, damp, tol, "graph")
    assert s.graph_error is None and s.graph_replays > 0, s.graph_error
    assert s._st == (2 if dtype == "complex128" else 1)
    assert s._cc_ready is (layout == "blockdiag")       # a BROADCAST c takes the unfused update + c.c
    assert ref["iiter"] == T and ref["istop"] == (2 if stop is None else 1)
    for mode in ("eager", "step", "show", "callback"):
        s, got = solve(Eop if mode == "eager" else Op, y, x0, damp, tol, mode)
        if mode == "eager":
            assert s.graph_replays == 0 and s.graph_error == "operator not on the graph-safe list"
        for f in FIELDS:
            np.testing.assert_array_equal(got[f], ref[f], err_msg=f"{mode}: {f}")
    assert "r2norm" in capsys.readouterr().out


def test_cgls_callback_sees_every_iteration(pm):
    from pylops_mpi_b200.optimization.cls_basic import CGLS
    Op, _, y, x0 = problem(pm, "float64", "blockdiag")
    seen = []
    x, istop, iiter, *_ = pm.cgls(Op, y, x0=x0, niter=12, tol=0.0, callback=lambda x: seen.append(host(x.asarray())))
    assert iiter == 12 and len(seen) == 12
    s = CGLS(Op)
    xs = s.setup(y=y, x0=x0, niter=12, tol=0.0)
    for got in seen:
        xs = s.step(xs)
        np.testing.assert_array_equal(got, host(xs.asarray()))
    np.testing.assert_array_equal(seen[-1], host(x.asarray()))
