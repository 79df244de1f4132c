"""Kirchhoff demigration in a velocity model: the eikonal traveltime solver (b2_eikonal_tables), the operator modes
``"eikonal"`` and ``"byot"`` of local.Kirchhoff / LSM, and their fixtures.

CPU: refshim's Jacobi restatement (tests/golden/refshim/pylops/waveeqprocessing/eikonal.py) against a heap-ordered
fast-marching solver of the same update and against closed-form traveltimes; refshim's byot branch; the fixtures of
tests/golden/kirchhoff_eikonal_golden.npz (made by make_golden_kirchhoff_eikonal.py: the reference's MPIVStack and
cgls over the restatement).  GPU: b2_eikonal_tables through the C ABI, bit for bit against the restatement, and the
operators through the public interface."""
import ctypes
import heapq
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_kirchhoff as mgk  # noqa: E402
import make_golden_kirchhoff_eikonal as mge  # noqa: E402
from op_checks import assert_cgls_replay_matches_steps, host  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "kirchhoff_eikonal_golden.npz"), allow_pickle=False)
KE, EK = mge.refshim_eikonal()
KREF, _ = mgk.refshim()
ARG, CONVERGE = 2002, 2007
SENT = 7.25
# cgls over 100 iterations magnifies rounding.  The fixture solve was rerun on the CPU with the sums reordered,
# everything else equal (make_golden_kirchhoff_eikonal.py --reorder): once with the spreading sums over image points
# descending, once with both the spreading and the stacking sums (over traces) descending.  Over P = 1, 2, 3 the cost
# history moved by up to 2.0e-2 (relative) and the model by up to 3.0e-3 of its largest value.  The tolerances are
# five times that spread, rounded up.
FLOW_COST_RTOL, FLOW_MINV_ATOL = 0.12, 1.5e-2
# the constant-velocity error bound  max(T - r / v) <= C h / v (1 + log(r / h)), C measured on the host over the
# grids of test_constant_velocity_error_bound (largest ratio 0.357 on the 3-D grid, 0.252 on the 81 x 60 one)
C_CONST = 0.36


def fmm(vel, spacing, node):
    """heap-ordered fast marching of refshim's Godunov update: nodes are accepted in increasing T, and a node's
    tentative value uses accepted neighbours only (others count as +inf)"""
    vel = np.asarray(vel, dtype=np.float64)
    shape = vel.shape
    h = np.asarray(spacing, dtype=np.float64)
    w = 1.0 / (h * h)
    slow = 1.0 / vel
    T = np.full(shape, np.inf)
    done = np.zeros(shape, dtype=bool)
    T[tuple(node)] = 0.0
    heap = [(0.0, tuple(node))]
    while heap:
        t, p = heapq.heappop(heap)
        if done[p]:
            continue
        done[p] = True
        for ax in range(3):
            for s in (-1, 1):
                q = list(p)
                q[ax] += s
                if not 0 <= q[ax] < shape[ax]:
                    continue
                q = tuple(q)
                if done[q]:
                    continue
                box = np.full((3, 3, 3), np.inf)
                for a2 in range(3):
                    for s2 in (-1, 1):
                        r = list(q)
                        r[a2] += s2
                        if 0 <= r[a2] < shape[a2] and done[tuple(r)]:
                            c = [1, 1, 1]
                            c[a2] += s2
                            box[tuple(c)] = T[tuple(r)]
                box[1, 1, 1] = np.inf
                nv = EK.godunov_step(box, np.full((3, 3, 3), slow[q]), h, w)[1, 1, 1]
                if nv < T[q]:
                    T[q] = nv
                    heapq.heappush(heap, (nv, q))
    return T


def jacobi1(vel, spacing, node):
    T, it = EK.jacobi(vel, spacing, [node])
    return T[0], it


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
def fixture_grids():
    z, x, t, srcs, recs, vel = mge.op_geometry(3)
    yield vel[None], EK.spacings((x, z)), EK.snap(srcs, (x, z))
    z, x, t, srcs, recs, vel, y = mge.op3_geometry(3)
    yield vel, EK.spacings((y, x, z)), EK.snap(srcs, (y, x, z))


@pytest.mark.parametrize("case", ["fixture-2d", "fixture-3d", "random-2d", "random-3d"])
def test_jacobi_reaches_the_fast_marching_solution(case):
    if case.startswith("fixture"):
        vel, h, nodes = list(fixture_grids())[case.endswith("3d")]
    else:
        rng = np.random.default_rng(3 if case == "random-2d" else 4)
        shape = (1, 23, 17) if case == "random-2d" else (7, 9, 8)
        grids = np.meshgrid(*[np.linspace(0, 1, n) for n in shape], indexing="ij")
        vel = 1500 + sum(rng.uniform(-300, 300) * np.sin(rng.uniform(1, 4) * g + rng.uniform(0, 6)) for g in grids)
        h = (2.5, 3.0, 4.0)
        nodes = np.stack([rng.integers(0, n, 3) for n in shape], axis=1)
    for node in nodes:
        Tj, _ = jacobi1(vel, h, node)
        Tf = fmm(vel, h, node)
        np.testing.assert_allclose(Tj, Tf, rtol=1e-12, atol=0)


def test_constant_velocity_error_bound():
    """T - r / v >= 0 (the scheme overestimates) and <= C h / v (1 + log(r / h)), r >= h"""
    v = 1000.0
    for shape, h, node in (((1, 81, 60), 4.0, (0, 10, 2)), ((1, 41, 41), 2.0, (0, 20, 20)),
                           ((9, 11, 10), 5.0, (4, 0, 9))):
        T, _ = jacobi1(np.full(shape, v), (h, h, h) if shape[0] > 1 else (1.0, h, h), node)
        idx = np.indices(shape).astype(np.float64)
        r = np.sqrt(sum(((i - c) * h) ** 2 for i, c in zip(idx, node)))
        err = T - r / v
        assert err.min() >= -1e-15
        m = r >= h
        assert np.all(err[m] <= C_CONST * h / v * (1 + np.log(r[m] / h)))


def test_refining_reduces_the_error():
    """the same physical points on grids h = 8, 4, 2 m: the worst error at those points falls with h"""
    v, L = 1000.0, 96.0
    errs = []
    for h in (8.0, 4.0, 2.0):
        n = int(L / h) + 1
        T, _ = jacobi1(np.full((1, n, n), v), (1.0, h, h), (0, 0, 0))
        k = int(16 / h)                                      # every 16 m
        X, Z = np.meshgrid(np.arange(0, n, k) * h, np.arange(0, n, k) * h, indexing="ij")
        errs.append(np.max(np.abs(T[0, ::k, ::k] - np.hypot(X, Z) / v)))
    assert errs[0] > errs[1] > errs[2]


def test_linear_gradient_error_shrinks_with_h():
    """v = v0 + k z: T = arccosh(1 + k^2 r^2 / (2 v_src v)) / k"""
    v0, k, L = 1000.0, 2.0, 96.0
    errs = []
    for h in (8.0, 4.0, 2.0):
        n = int(L / h) + 1
        z = np.arange(n) * h
        vel = np.broadcast_to(v0 + k * z, (1, n, n)).copy()
        src = (0, n // 2, 0)
        T, _ = jacobi1(vel, (1.0, h, h), src)
        X, Z = np.meshgrid(np.arange(n) * h, z, indexing="ij")
        r2 = (X - src[1] * h) ** 2 + Z ** 2
        exact = np.arccosh(1 + k * k * r2 / (2 * v0 * (v0 + k * Z))) / k
        s = int(16 / h)
        errs.append(np.max(np.abs(T[0] - exact)[::s, ::s]))
    assert errs[0] > errs[1] > errs[2]


def test_refshim_byot_with_analytic_tables_is_the_analytic_restatement():
    z, x, t, srcs, recs, vel = mgk.op_geometry(2)
    h, off = mgk.wavelet("ricker21")
    A = KREF.Kirchhoff(z, x, t, srcs, recs, vel, h, off, mode="analytic")
    B = KE.Kirchhoff(z, x, t, srcs, recs, None, h, off, mode="byot", trav=(A.trav_srcs, A.trav_recs))
    rng = np.random.default_rng(2)
    m, d = rng.standard_normal(A.shape[1]), rng.standard_normal(A.shape[0])
    np.testing.assert_array_equal(A._matvec(m), B._matvec(m))
    np.testing.assert_array_equal(A._rmatvec(d), B._rmatvec(d))


def test_fixture_inventory_and_geometry():
    keys = set(GOLD.files)
    for tag in ("op", "op3"):
        for P in (1, 2, 3):
            for w in mgk.WAVELETS:
                assert {f"{tag}/P{P}/{w}/y", f"{tag}/P{P}/{w}/ya"} <= keys
    for P in (1, 2, 3):
        assert {f"flow/P{P}/{k}" for k in ("madj", "minv", "iiter", "cost")} <= keys
    assert os.path.getsize(os.path.join(HERE, "golden", "kirchhoff_eikonal_golden.npz")) < 1_000_000
    mge.check_cases()                                   # distance from integers, record ends, Manhattan extent


@pytest.mark.parametrize("tag", ["op", "op3"])
@pytest.mark.parametrize("wav", mgk.WAVELETS)
def test_fixtures_follow_the_restatement(tag, wav):
    """P = 1: one operator, the fixture is its forward and adjoint"""
    h, off = mgk.wavelet(wav)
    if tag == "op":
        (z, x, t, srcs, recs, vel), y = mge.op_geometry(1), None
    else:
        z, x, t, srcs, recs, vel, y = mge.op3_geometry(1)
    Op = KE.Kirchhoff(z, x, t, srcs, recs, vel, h, off, y=y, mode="eikonal")
    m, d = mge.op_inputs(1, tag == "op3")
    gy, gya = GOLD[f"{tag}/P1/{wav}/y"], GOLD[f"{tag}/P1/{wav}/ya"]
    np.testing.assert_allclose(Op._matvec(m), gy, rtol=0, atol=1e-12 * np.abs(gy).max())
    np.testing.assert_allclose(Op._rmatvec(d), gya, rtol=0, atol=1e-12 * np.abs(gya).max())


# ---------------------------------------------------------------------------------------------------------------
# GPU: b2_eikonal_tables through the C ABI
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


def dev(a):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def c_eikonal(pm, vel, shape, h, nodes, max_iter, table_ptr, info=None, work=None):
    import torch
    L = pm._lib
    nodes = np.ascontiguousarray(nodes, dtype=np.int64).reshape(-1, 3)
    if work is None:
        work = torch.empty(max(8, L.lib.b2_eikonal_work_bytes(*shape, max(1, len(nodes)))), dtype=torch.uint8,
                           device="cuda")
    rc = L.lib.b2_eikonal_tables(L.ctx(), vel.data_ptr() if vel is not None else None, *shape, *h,
                                 nodes.ctypes.data if len(nodes) else None, len(nodes), max_iter, table_ptr,
                                 work.data_ptr() if work is not None else None, info, L.stream())
    torch.cuda.synchronize()
    return rc


def device_tables(pm, vel, h, nodes, max_iter=None, guard=3):
    """b2_eikonal_tables into a guarded buffer: (tables (n, ny, nx, nz), info, rc)"""
    import torch
    shape = vel.shape
    n, ni = len(nodes), int(np.prod(shape))
    b = torch.full((n * ni + 2 * guard + 1,), SENT, dtype=torch.float64, device="cuda")
    t = b[guard + 1:guard + 1 + n * ni]
    info = (ctypes.c_longlong * 4)()
    rc = c_eikonal(pm, dev(vel), shape, h, nodes, max_iter or ni, t.data_ptr(), info)
    hb = host(b)
    assert np.all(hb[:guard + 1] == SENT) and np.all(hb[guard + 1 + n * ni:] == SENT)
    return host(t).reshape((n,) + shape), list(info), rc


def lens(shape, seed=0):
    """a vertical gradient times a slow lens on an index grid"""
    idx = np.indices(shape).astype(np.float64)
    c = [(n - 1) / 2 for n in shape]
    r2 = sum(((i - cc) / max(n / 4, 1)) ** 2 for i, cc, n in zip(idx, c, shape))
    return (900.0 + 25.0 * idx[-1]) * (1 - 0.4 * np.exp(-r2)) * (1 + 0.02 * np.random.default_rng(seed).random(shape))


def corners(shape):
    return [(a, b, c) for a in (0, shape[0] - 1) for b in (0, shape[1] - 1) for c in (0, shape[2] - 1)]


SOLVER_CASES = {
    # name: (shape, spacings (dy, dx, dz), nodes)
    "2d-lens-corners": ((1, 45, 37), (1.0, 4.0, 3.0), corners((1, 45, 37)) + [(0, 22, 18)]),
    "2d-exact-tile": ((1, 32, 32), (1.0, 2.0, 5.0), [(0, 31, 0)]),
    "2d-tutorial": ((1, 81, 60), (1.0, 4.0, 4.0), [(0, 10, 2), (0, 40, 5), (0, 70, 2)]),
    "3d-small": ((3, 5, 4), (3.0, 4.0, 2.5), corners((3, 5, 4))),
    "3d-ny2": ((2, 9, 11), (1.5, 2.0, 2.5), [(0, 0, 0), (1, 8, 10), (1, 4, 5)]),
    "3d-lens-corners": ((11, 13, 17), (3.0, 4.0, 2.5), corners((11, 13, 17))[:5]),
    "3d-mid": ((27, 41, 35), (4.0, 3.0, 5.0), [(0, 0, 0), (26, 40, 34), (13, 20, 3), (5, 37, 30), (20, 2, 17)]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SOLVER_CASES))
def test_eikonal_tables_equal_numpy_bitwise(pm, name):
    shape, h, nodes = SOLVER_CASES[name]
    vel = lens(shape, seed=len(name))
    T, info, rc = device_tables(pm, vel, h, nodes)
    assert rc == 0
    R, iters = EK.jacobi(vel, h, nodes)
    np.testing.assert_array_equal(T, R)
    assert info[0] == iters
    assert info[1] >= 1 and 0 < info[2] <= info[3]


@pytest.mark.gpu
def test_eikonal_tables_repeat_bitwise(pm):
    shape, h, nodes = SOLVER_CASES["3d-lens-corners"]
    vel = lens(shape)
    a, _, _ = device_tables(pm, vel, h, nodes)
    b, _, _ = device_tables(pm, vel, h, nodes)
    assert a.tobytes() == b.tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("max_iter", [1, 5, 9])
def test_eikonal_tables_not_converged(pm, max_iter):
    """max_iter below the fixed point: B2_ERR_CONVERGE, and the table holds the max_iter-th iterate"""
    for shape, h in (((1, 40, 30), (1.0, 2.0, 3.0)), ((9, 10, 11), (2.0, 3.0, 4.0))):
        vel = lens(shape)
        nodes = [(0, 0, 0), (shape[0] - 1, shape[1] // 2, shape[2] - 1)]
        T, info, rc = device_tables(pm, vel, h, nodes, max_iter=max_iter)
        assert rc == CONVERGE
        R, iters = EK.jacobi(vel, h, nodes, max_iter=max_iter)
        assert iters == max_iter
        np.testing.assert_array_equal(T, R)


@pytest.mark.gpu
def test_eikonal_tables_error_codes_leave_table_untouched(pm):
    import torch
    shape, h, nodes = (2, 6, 5), (1.0, 2.0, 3.0), [(0, 0, 0), (1, 5, 4)]
    vel = lens(shape)
    ni = int(np.prod(shape))
    table = torch.full((2 * ni,), SENT, dtype=torch.float64, device="cuda")
    dv = dev(vel)
    work = torch.empty(pm._lib.lib.b2_eikonal_work_bytes(*shape, 2), dtype=torch.uint8, device="cuda")
    tp = table.data_ptr()
    bad = [
        dict(vel=None), dict(table=None), dict(work=None), dict(nodes=np.zeros((0, 3))), dict(max_iter=0),
        dict(shape=(0, 6, 5)), dict(shape=(2, 0, 5)), dict(nodes=[(0, 0, 0), (2, 5, 4)]),
        dict(nodes=[(0, 0, 0), (1, 6, 4)]), dict(nodes=[(0, 0, -1), (1, 5, 4)]), dict(h=(0.0, 2.0, 3.0)),
        dict(h=(1.0, -2.0, 3.0)), dict(h=(1.0, 2.0, np.inf)), dict(h=(1.0, np.nan, 3.0)),
        dict(vel=dev(np.where(np.arange(ni).reshape(shape) == 7, 0.0, vel))),
        dict(vel=dev(np.where(np.arange(ni).reshape(shape) == 3, np.nan, vel))),
        dict(vel=dev(np.where(np.arange(ni).reshape(shape) == 0, -5.0, vel))),
        dict(vel=dev(np.where(np.arange(ni).reshape(shape) == 9, np.inf, vel))),
    ]
    for kw in bad:
        a = dict(vel=dv, shape=shape, h=h, nodes=nodes, max_iter=ni, table=tp, work=work)
        a.update(kw)
        L = pm._lib
        nd = np.ascontiguousarray(np.asarray(a["nodes"], dtype=np.int64).reshape(-1, 3))
        rc = L.lib.b2_eikonal_tables(L.ctx(), a["vel"].data_ptr() if a["vel"] is not None else None, *a["shape"],
                                     *a["h"], nd.ctypes.data if len(nd) else None, len(nd), a["max_iter"],
                                     a["table"], a["work"].data_ptr() if a["work"] is not None else None, None,
                                     L.stream())
        torch.cuda.synchronize()
        assert rc == ARG, kw
        assert torch.all(table == SENT), kw
    assert pm._lib.lib.b2_eikonal_work_bytes(0, 3, 3, 1) == 0
    assert pm._lib.lib.b2_eikonal_work_bytes(3, 3, 3, 0) == 0


# ---------------------------------------------------------------------------------------------------------------
# GPU: the operators
# ---------------------------------------------------------------------------------------------------------------
def geometry(tag, P, rank):
    if tag == "op":
        return mge.op_geometry(P, rank) + (None,)
    return mge.op3_geometry(P, rank)


def op_vstack(pm, tag, P, wav, dtype="float64"):
    h, off = mgk.wavelet(wav)
    ops = []
    for r in range(P):
        z, x, t, srcs, recs, vel, y = geometry(tag, P, r)
        ops.append(pm.local.Kirchhoff(z, x, t, srcs, recs, vel, h, off, y=y, mode="eikonal", dtype=dtype))
    return pm.MPIVStack(ops)


def bcast(pm, a):
    return pm.DistributedArray.to_dist(a, partition=pm.Partition.BROADCAST)


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["op", "op3"])
def test_operator_tables_equal_the_restatement(pm, tag):
    z, x, t, srcs, recs, vel, y = geometry(tag, 3, None)
    h, off = mgk.wavelet("spike")
    K = pm.local.Kirchhoff(z, x, t, srcs, recs, vel, h, off, y=y, mode="eikonal")
    ts, tr = KE.traveltime_tables(z, x, srcs, recs, vel, y=y)
    assert K.trav_srcs.shape == ts.shape and K.trav_recs.shape == tr.shape
    np.testing.assert_array_equal(host(K.trav_srcs), ts)
    np.testing.assert_array_equal(host(K.trav_recs), tr)


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["op", "op3"])
@pytest.mark.parametrize("P", [1, 2, 3])
@pytest.mark.parametrize("wav", mgk.WAVELETS)
def test_operator_vs_reference_fixtures(pm, tag, P, wav):
    Op = op_vstack(pm, tag, P, wav)
    m, d = mge.op_inputs(P, tag == "op3")
    y = host((Op @ bcast(pm, m)).asarray())
    ya = host((Op.H @ pm.DistributedArray.to_dist(d)).asarray())
    gy, gya = GOLD[f"{tag}/P{P}/{wav}/y"], GOLD[f"{tag}/P{P}/{wav}/ya"]
    np.testing.assert_allclose(y, gy, rtol=0, atol=1e-12 * np.abs(gy).max())
    if wav == "spike" and P == 1:
        np.testing.assert_array_equal(ya, gya)            # identity convolution, one rank: pylops' stacking exactly
    else:
        np.testing.assert_allclose(ya, gya, rtol=0, atol=1e-12 * np.abs(gya).max())


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["op", "op3"])
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_operator_dottest(pm, tag, dtype):
    Op = op_vstack(pm, tag, 2, "ricker21", dtype)
    rng = np.random.default_rng(5)
    u = bcast(pm, rng.standard_normal(Op.shape[1]).astype(dtype))
    v = pm.DistributedArray.to_dist(rng.standard_normal(Op.shape[0]).astype(dtype))
    assert pm.dottest(Op, u, v, rtol=1e-4 if dtype == "float32" else 1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["op", "op3"])
def test_byot_round_trip_bitwise(pm, tag):
    import torch
    z, x, t, srcs, recs, vel, y = geometry(tag, 2, None)
    h, off = mgk.wavelet("asym/o4")
    K = pm.local.Kirchhoff(z, x, t, srcs, recs, vel, h, off, y=y, mode="eikonal")
    B = pm.local.Kirchhoff(z, x, t, srcs, recs, None, h, off, y=y, mode="byot", trav=(K.trav_srcs, K.trav_recs))
    Bn = pm.local.Kirchhoff(z, x, t, srcs, recs, 3.0, h, off, y=y, mode="byot",
                            trav=(host(K.trav_srcs), host(K.trav_recs).astype(np.float64)))
    assert torch.equal(B._ts, K._ts) and torch.equal(Bn._tr, K._tr)
    rng = np.random.default_rng(6)
    for dt in (torch.float64, torch.float32):
        m = torch.as_tensor(rng.standard_normal(K.shape[1])).to(dt).cuda()
        d = torch.as_tensor(rng.standard_normal(K.shape[0])).to(dt).cuda()
        for Op in (B, Bn):
            assert torch.equal(Op.matvec(m), K.matvec(m))
            assert torch.equal(Op.rmatvec(d), K.rmatvec(d))
    # float32 user tables are converted once: the operator uses exactly their float64 values
    B32 = pm.local.Kirchhoff(z, x, t, srcs, recs, None, h, off, y=y, mode="byot",
                             trav=(K.trav_srcs.float(), host(K.trav_recs).astype(np.float32)))
    assert torch.equal(B32.trav_srcs, K.trav_srcs.float().double())


@pytest.mark.gpu
def test_lsm_pass_through_and_graph_replay(pm):
    z, x, t, srcs, recs, vel = mge.op_geometry(2)
    h, off = mgk.wavelet("ricker21")
    lsm = pm.local.LSM(z, x, t, srcs, recs, vel, h, off, mode="eikonal", dtype="float32")
    assert lsm.Demop.mode == "eikonal" and lsm.Demop.dtype == np.float32
    Op = op_vstack(pm, "op", 2, "ricker21")
    rng = np.random.default_rng(12)
    yv = Op @ bcast(pm, rng.standard_normal(Op.shape[1]))
    assert_cgls_replay_matches_steps(pm, Op, yv, bcast(pm, np.zeros(Op.shape[1])), 25, 20)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
def test_flow_vs_reference(pm, P):
    ops = []
    for r in range(P):
        z, x, t, srcs, recs, vel, wav, wavc, refl = mge.flow_setup(P, r)
        ops.append(pm.local.LSM(z, x, t, srcs, recs, vel, wav, wavc, mode="eikonal").Demop)
    V = pm.MPIVStack(ops)
    d = V @ bcast(pm, refl.ravel())
    madj = host((V.H @ d).asarray())
    minv, _, iiter, _, _, cost = pm.cgls(V, d, x0=bcast(pm, np.zeros(V.shape[1])), niter=mge.FLOW_NITER)
    g = f"flow/P{P}"
    gm, gi = GOLD[f"{g}/madj"], GOLD[f"{g}/minv"]
    np.testing.assert_allclose(madj, gm, rtol=0, atol=1e-12 * np.abs(gm).max())
    assert int(iiter) == int(GOLD[f"{g}/iiter"])
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"{g}/cost"], rtol=FLOW_COST_RTOL)
    np.testing.assert_allclose(host(minv.asarray()), gi, rtol=0, atol=FLOW_MINV_ATOL * np.abs(gi).max())


@pytest.mark.gpu
def test_operator_argument_errors_eikonal_byot(pm, monkeypatch):
    import torch
    z, x, t, srcs, recs, vel = mge.op_geometry(1)
    h = np.ones(3)
    K = pm.local.Kirchhoff
    with pytest.raises(NotImplementedError, match="mode"):
        K(z, x, t, srcs, recs, 1000.0, h, 1, mode="eikonal")
    with pytest.raises(NotImplementedError, match="mode"):
        K(z, x, t, srcs, recs, vel, h, 1, mode="byot")
    with pytest.raises(NotImplementedError, match="trav"):
        K(z, x, t, srcs, recs, vel, h, 1, mode="eikonal", trav=(np.zeros(2), np.zeros(2)))
    ni, ns, nr = x.size * z.size, srcs.shape[1], recs.shape[1]
    with pytest.raises(NotImplementedError, match="trav"):
        K(z, x, t, srcs, recs, None, h, 1, mode="byot", trav=np.zeros((ni, ns * nr)))
    for trav in ((np.zeros((ni, ns + 1)), np.zeros((ni, nr))), (np.zeros((ni, ns)), np.zeros((ni - 1, nr))),
                 (np.zeros((ni, ns), dtype=complex), np.zeros((ni, nr))), (np.zeros(ni), np.zeros((ni, nr)))):
        with pytest.raises(ValueError):
            K(z, x, t, srcs, recs, None, h, 1, mode="byot", trav=trav)
    for bad in (vel[:-1], vel.T, np.where(vel > 1000, 0.0, vel), np.where(vel > 1000, np.nan, vel),
                np.where(vel > 1000, -vel, vel), np.where(vel > 1000, np.inf, vel), vel.astype(complex)):
        with pytest.raises(ValueError):
            K(z, x, t, srcs, recs, bad, h, 1, mode="eikonal")
    xs = x.copy()
    xs[3] += 0.5
    with pytest.raises(ValueError, match="uniform"):
        K(z, xs, t, srcs, recs, vel, h, 1, mode="eikonal")
    for s in (np.vstack(([x[-1] + 2.5], [4.0])), np.vstack(([-2.5], [4.0])), np.vstack(([4.0], [z[-1] + 1.6]))):
        with pytest.raises(ValueError, match="outside"):
            K(z, x, t, s, recs, vel, h, 1, mode="eikonal")
    K(z, x, t, np.vstack(([x[-1] + 1.9], [4.0])), recs, vel, h, 1, mode="eikonal")   # snaps onto the last node
    # any real dtype of vel; a torch tensor too
    a = K(z, x, t, srcs, recs, vel.astype(np.float32), h, 1, mode="eikonal")
    b = K(z, x, t, srcs, recs, torch.as_tensor(vel.astype(np.float32)), h, 1, mode="eikonal")
    assert torch.equal(a._ts, b._ts)
    c = K(z, x, t, srcs, recs, np.full(vel.shape, 1000, dtype=np.int32), h, 1, mode="eikonal")
    assert c.trav_srcs.dtype == torch.float64
    # the budget: tables (and the solver's work buffer) must fit
    table_bytes = (ns + nr) * ni * 8
    monkeypatch.setattr(pm.local, "KIRCHHOFF_TABLE_BYTES", table_bytes - 8)
    with pytest.raises(ValueError, match=str(table_bytes)):
        K(z, x, t, srcs, recs, None, h, 1, mode="byot", trav=(np.zeros((ni, ns)), np.zeros((ni, nr))))
    with pytest.raises(ValueError, match="KIRCHHOFF_TABLE_BYTES"):
        K(z, x, t, srcs, recs, vel, h, 1, mode="eikonal")
    monkeypatch.setattr(pm.local, "KIRCHHOFF_TABLE_BYTES", table_bytes)
    K(z, x, t, srcs, recs, None, h, 1, mode="byot", trav=(np.zeros((ni, ns)), np.zeros((ni, nr))))
    with pytest.raises(ValueError, match="work buffer"):
        K(z, x, t, srcs, recs, vel, h, 1, mode="eikonal")
    # one point per solve still fits: the same tables as without a budget
    one = table_bytes + pm._lib.lib.b2_eikonal_work_bytes(1, x.size, z.size, 1)
    monkeypatch.setattr(pm.local, "KIRCHHOFF_TABLE_BYTES", one)
    small = K(z, x, t, srcs, recs, vel, h, 1, mode="eikonal")
    monkeypatch.undo()
    full = K(z, x, t, srcs, recs, vel, h, 1, mode="eikonal")
    assert torch.equal(small._ts, full._ts) and torch.equal(small._tr, full._tr)
    # a chunked analytic operator has no resident tables
    monkeypatch.setattr(pm.local, "KIRCHHOFF_TABLE_BYTES", (ns + nr) * 8 * 32)
    ch = K(z, x, t, srcs, recs, 1000.0, h, 1, mode="analytic")
    assert ch.chunked
    with pytest.raises(AttributeError):
        ch.trav_srcs
    with pytest.raises(AttributeError):
        ch.trav_recs
