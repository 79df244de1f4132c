"""3-D Kirchhoff demigration (pylops.waveeqprocessing.Kirchhoff / LSM with a ``y`` axis inside MPIVStack), the
device traveltime tables and the chunked apply.

CPU: refshim's 3-D restatement against tables and dense matrices built point by point from the definition, the host
tables of ``local`` against the restatement's, and the fixtures of tests/golden/kirchhoff3d_golden.npz (made by
make_golden_kirchhoff3d.py: the reference's MPIVStack and cgls over the restatement).  GPU: b2_kirchhoff_tables and
b2_kirchhoff_chunk through the C ABI (bit for bit against NumPy and against one b2_kirchhoff call), and the 3-D and
chunked operators through the public interface."""
import math
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_kirchhoff as mgk  # noqa: E402
import make_golden_kirchhoff3d as m3  # noqa: E402
from op_checks import assert_cgls_replay_matches_steps, host, needs_gpus, run_on_ranks  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "kirchhoff3d_golden.npz"), allow_pickle=False)
KREF, _ = mgk.refshim()
KREF3 = m3.refshim3d()
U32 = 2.0 ** -24
ARG, DT = 2002, 2001
SENT = 7.25
# cgls over 30 iterations magnifies rounding.  The fixture solve was run twice more on the CPU with the sums
# reordered, everything else equal: once with the spreading sums over image points descending, once with both the
# spreading and the stacking sums (over traces) descending.  Over P = 1, 2, 3 the cost history moved by up to 1.02e-1
# (relative) and the model by up to 3.9e-3 of its largest value.  The tolerances are five times that spread.
FLOW_COST_RTOL, FLOW_MINV_ATOL = 0.55, 2e-2


# ---------------------------------------------------------------------------------------------------------------
# the definition, point by point
# ---------------------------------------------------------------------------------------------------------------
def tables_by_definition(z, x, y, srcs, recs, vel):
    """(ni, n) tables from scalar IEEE float64 arithmetic: dist2 = (x - px)^2 + (z - pz)^2, then + (y - py)^2"""
    def table(pts):
        out = []
        for yy in y:
            for xx in x:
                for zz in z:
                    row = []
                    for py, px, pz in pts.T:
                        dx, dz, dy = float(xx) - float(px), float(zz) - float(pz), float(yy) - float(py)
                        dist2 = dx * dx + dz * dz
                        dist2 += dy * dy
                        row.append(math.sqrt(dist2) / float(vel))
                    out.append(row)
        return np.array(out)
    return table(srcs), table(recs)


def spread_matrix(ts, tr, dt, nt):
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


def op_matrix(ts, tr, dt, nt, h, off):
    C = np.zeros((nt, nt))
    for i in range(nt):
        for j in range(nt):
            if 0 <= i + off - j < len(h):
                C[i, j] = h[i + off - j]
    return np.kron(np.eye(ts.shape[1] * tr.shape[1]), C) @ spread_matrix(ts, tr, dt, nt)


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wav", mgk.WAVELETS)
def test_refshim_3d_is_the_dense_definition(wav):
    z, x, t, srcs, recs, vel, y = m3.op_geometry(2)
    h, off = mgk.wavelet(wav)
    Op = KREF3.Kirchhoff(z, x, t, srcs, recs, vel, h, off, y=y, mode="analytic")
    assert Op.dims == (m3.OP_NY, m3.OP_NX, m3.OP_NZ)
    assert Op.shape == (srcs.shape[1] * recs.shape[1] * t.size, y.size * x.size * z.size)
    ts, tr = tables_by_definition(z, x, y, srcs, recs, vel)
    np.testing.assert_array_equal(Op.trav_srcs, ts)
    np.testing.assert_array_equal(Op.trav_recs, tr)
    M = op_matrix(ts, tr, Op.dt, t.size, h, off)
    rng = np.random.default_rng(3)
    m, d = rng.standard_normal(Op.shape[1]), rng.standard_normal(Op.shape[0])
    scale = np.abs(M).sum() + 1
    np.testing.assert_allclose(Op.matvec(m), M @ m, rtol=0, atol=1e-13 * scale)
    np.testing.assert_allclose(Op.rmatvec(d), M.T @ d, rtol=0, atol=1e-13 * scale)


def test_refshim_3d_module_without_y_is_the_2d_restatement():
    z, x, t, srcs, recs, vel = mgk.op_geometry(2)
    h, off = mgk.wavelet("asym/o4")
    a = KREF3.Kirchhoff(z, x, t, srcs, recs, vel, h, off, mode="analytic")
    b = KREF.Kirchhoff(z, x, t, srcs, recs, vel, h, off, mode="analytic")
    assert a.dims == b.dims and a.shape == b.shape
    np.testing.assert_array_equal(a.trav_srcs, b.trav_srcs)
    np.testing.assert_array_equal(a.trav_recs, b.trav_recs)
    m, d = mgk.op_inputs(2)
    n = a.shape[0]
    np.testing.assert_array_equal(a.matvec(m), b.matvec(m))
    np.testing.assert_array_equal(a.rmatvec(d[:n]), b.rmatvec(d[:n]))


@pytest.mark.parametrize("geom", ["op", "flow"])
def test_local_tables_3d_equal_the_restatement(geom):
    from pylops_mpi_b200.local import _traveltime_tables
    if geom == "op":
        z, x, t, srcs, recs, vel, y = m3.op_geometry(3)
    else:
        z, x, t, srcs, recs, vel, *_, y = m3.flow_setup(2, 1)
    a = _traveltime_tables(z, x, srcs, recs, vel, y=y)
    b = KREF3.traveltime_tables(z, x, srcs, recs, vel, y=y)
    for u, v in zip(a, b):
        assert u.dtype == np.float64 and u.shape == v.shape == (y.size * x.size * z.size, u.shape[1])
        np.testing.assert_array_equal(u, v)


def test_kirchhoff3d_fixture_inventory():
    names = set()
    for P in (1, 2, 3):
        for wav in mgk.WAVELETS:
            y, ya = GOLD[f"{mgk.key(P, wav)}/y"], GOLD[f"{mgk.key(P, wav)}/ya"]
            assert y.dtype == np.float64 and y.shape == (P * m3.OP_NS * m3.OP_NR * m3.OP_NT,)
            assert ya.dtype == np.float64 and ya.shape == (m3.OP_NY * m3.OP_NX * m3.OP_NZ,)
            names |= {f"{mgk.key(P, wav)}/y", f"{mgk.key(P, wav)}/ya"}
        for k in ("madj", "minv", "iiter", "cost"):
            names.add(f"flow/P{P}/{k}")
        assert int(GOLD[f"flow/P{P}/iiter"]) == m3.FLOW_NITER
        assert GOLD[f"flow/P{P}/cost"].shape == (m3.FLOW_NITER + 1,)
        ni = m3.FLOW_NY * m3.FLOW_NX * m3.FLOW_NZ
        assert GOLD[f"flow/P{P}/minv"].shape == GOLD[f"flow/P{P}/madj"].shape == (ni,)
    assert sorted(GOLD.files) == sorted(names)
    assert os.path.getsize(os.path.join(HERE, "golden", "kirchhoff3d_golden.npz")) < 400_000


@pytest.mark.parametrize("P", [1, 2, 3])
@pytest.mark.parametrize("wav", mgk.WAVELETS)
def test_kirchhoff3d_fixtures_follow_the_definition(P, wav):
    z, x, t, srcs, recs, vel, y = m3.op_geometry(P)
    ts, tr = tables_by_definition(z, x, y, srcs, recs, vel)
    h, off = mgk.wavelet(wav)
    M = op_matrix(ts, tr, m3.OP_DT, m3.OP_NT, h, off)
    m, d = m3.op_inputs(P)
    gy, gya = GOLD[f"{mgk.key(P, wav)}/y"], GOLD[f"{mgk.key(P, wav)}/ya"]
    np.testing.assert_allclose(gy, M @ m, rtol=0, atol=1e-13 * np.abs(gy).max())
    np.testing.assert_allclose(gya, M.T @ d, rtol=0, atol=1e-13 * np.abs(gya).max())


@pytest.mark.parametrize("P", [1, 3])
def test_kirchhoff3d_flow_fixture_madj_follows_the_restatement(P):
    z, x, t, srcs, recs, v0, wav, wavc, refl, y = m3.flow_setup(P)
    Op = KREF3.Kirchhoff(z, x, t, srcs, recs, v0, wav, wavc, y=y, mode="analytic")
    madj = Op.rmatvec(Op.matvec(refl.ravel()))
    np.testing.assert_allclose(GOLD[f"flow/P{P}/madj"], madj, rtol=0, atol=1e-12 * np.abs(madj).max())


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernels through the C ABI
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


def dev(a):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def guarded(n, dtype, guard=3):
    """(buffer of n + 2 * guard + 1 sentinels, the view at an odd element offset that receives the output)"""
    import torch
    b = torch.full((n + 2 * guard + 1,), SENT, dtype=dtype, device="cuda")
    return b, b[guard + 1:guard + 1 + n]


def guards_intact(b, n, guard=3):
    h = host(b)
    return bool(np.all(h[:guard + 1] == SENT) and np.all(h[guard + 1 + n:] == SENT))


def c_tables(pm, ay, ax, az, ny, nx, nz, pts, n, vel, i0, nc, table):
    L = pm._lib
    return L.lib.b2_kirchhoff_tables(L.ctx(), ay, ax, az, ny, nx, nz, pts, n, vel, i0, nc, table, L.stream())


def device_table(pm, z, x, pts, vel, y, i0, nc):
    """b2_kirchhoff_tables for image points [i0, i0 + nc) into a guarded buffer: the (n, nc) table"""
    import torch
    n = pts.shape[1]
    ay, ax, az, dp = (None if y is None else dev(y)), dev(x), dev(z), dev(pts)
    b, t = guarded(n * nc, torch.float64)
    rc = c_tables(pm, None if ay is None else ay.data_ptr(), ax.data_ptr(), az.data_ptr(), 0 if y is None else len(y),
                  len(x), len(z), dp.data_ptr(), n, float(vel), i0, nc, t.data_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    assert guards_intact(b, n * nc)
    return host(t).reshape(n, nc)


def table_geometry(name):
    """(z, x, srcs, recs, vel, y) of a table case"""
    if name == "tutorial-2d":
        z, x, t, srcs, recs, vel, *_ = mgk.flow_setup(1)          # integer axes, np.arange(nx) * 4
        return z, x, srcs, recs, vel, None
    if name == "op-2d":
        z, x, t, srcs, recs, vel = mgk.op_geometry(3)
        return z, x, srcs, recs, vel, None
    if name == "op-3d":
        z, x, t, srcs, recs, vel, y = m3.op_geometry(3)           # sources on grid points
        return z, x, srcs, recs, vel, y
    if name == "flow-3d":
        z, x, t, srcs, recs, vel, *_, y = m3.flow_setup(3)
        return z, x, srcs, recs, vel, y
    rng = np.random.default_rng(17)
    y, x, z = np.linspace(-30.5, 12.25, 7), np.arange(-5, 6) * 3.3, np.linspace(-2.0, 40.7, 9)
    pts = np.vstack((rng.uniform(-40, 20, 6), rng.uniform(-20, 20, 6), rng.uniform(-5, 45, 6)))
    pts[:, 0] = (y[2], x[0], z[4])                                # one point exactly on the grid: trav = 0
    if name == "negative-2d":
        return z, x, pts[1:, :3], pts[1:, 3:], 1487.3, None
    return z, x, pts[:, :3], pts[:, 3:], 1487.3, y                # negative-3d


TABLE_CASES = ["tutorial-2d", "op-2d", "op-3d", "flow-3d", "negative-2d", "negative-3d"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", TABLE_CASES)
def test_device_tables_equal_numpy_bitwise(pm, name):
    """whole image and chunks of 96 points (ni is not a multiple of 32 in any case, so the last chunk is short),
    and chunks starting off a multiple of 32"""
    from pylops_mpi_b200.local import _traveltime_tables
    z, x, srcs, recs, vel, y = table_geometry(name)
    ni = (1 if y is None else len(y)) * len(x) * len(z)
    assert ni % 32 != 0
    for pts, ref in zip((srcs, recs), _traveltime_tables(z, x, srcs, recs, vel, y=y)):
        ref = ref.T                                               # (n, ni)
        np.testing.assert_array_equal(device_table(pm, z, x, pts, vel, y, 0, ni), ref)
        for i0 in list(range(0, ni, 96)) + [5, ni - 7]:
            nc = min(96, ni - i0)
            np.testing.assert_array_equal(device_table(pm, z, x, pts, vel, y, i0, nc), ref[:, i0:i0 + nc])


def random_tables(ni, ns, nr, nt, dt, seed):
    """(ni, ns), (ni, nr) float64 tables whose pairs cover [0, nt + 3) samples, some at trav = 0 and on nt - 2"""
    rng = np.random.default_rng(seed)
    ts = rng.uniform(0, (nt + 3) * dt / 2, (ni, ns))
    tr = rng.uniform(0, (nt + 3) * dt / 2, (ni, nr))
    ts[0], tr[0] = 0.0, 0.0
    ts[1], tr[1] = (nt - 2) * dt / 2, (nt - 2) * dt / 2
    return ts, tr


def c_chunk(pm, x, y, ts, tr, ni, i0, nc, ns, nr, nt, dt, adjoint, accumulate, code):
    L = pm._lib
    return L.lib.b2_kirchhoff_chunk(L.ctx(), x, y, ts, tr, ni, i0, nc, ns, nr, nt, dt, adjoint, accumulate, code,
                                    L.stream())


def chunked_vs_one_call(pm, ni, ns, nr, nt, dtype, bounds, seed):
    import torch
    tdt = {np.float32: torch.float32, np.float64: torch.float64}[dtype]
    code = pm._lib.F32 if dtype == np.float32 else pm._lib.F64
    dt = 0.004
    ts, tr = random_tables(ni, ns, nr, nt, dt, seed)
    rng = np.random.default_rng(seed + 1)
    L = pm._lib
    tsd, trd = dev(ts.T), dev(tr.T)
    for adjoint in (0, 1):
        nin, nout = (ns * nr * nt, ni) if adjoint else (ni, ns * nr * nt)
        x = torch.as_tensor(rng.standard_normal(nin).astype(dtype)).cuda()
        ref = torch.empty(nout, dtype=tdt, device="cuda")
        assert L.lib.b2_kirchhoff(L.ctx(), x.data_ptr(), ref.data_ptr(), tsd.data_ptr(), trd.data_ptr(), ni, ns, nr,
                                  nt, dt, adjoint, code, L.stream()) == 0
        b, out = guarded(nout, tdt)
        edges = [0] + list(bounds) + [ni]
        for a, e in zip(edges[:-1], edges[1:]):
            cts, ctr = dev(ts[a:e].T), dev(tr[a:e].T)
            rc = c_chunk(pm, x.data_ptr(), out.data_ptr(), cts.data_ptr(), ctr.data_ptr(), ni, a, e - a, ns, nr, nt,
                         dt, adjoint, int(a > 0 and not adjoint), code)
            assert rc == 0, (a, e, rc)
        torch.cuda.synchronize()
        assert guards_intact(b, nout)
        assert torch.equal(out, ref), (adjoint, bounds, (out - ref).abs().max().item())


# (ni, ns, nr, nt): traces in shared memory, and traces past it (float64 nt > 1472, float32 nt > 2944)
CHUNK_SHAPES = {"smem": (250, 3, 4, 20), "global": (150, 2, 3, 3000)}
SPLITS = [(32,), (64, 96), (32, 64, 96, 128, 224), (224,)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("path", list(CHUNK_SHAPES))
def test_chunked_apply_equals_one_call_bitwise(pm, dtype, path):
    ni, ns, nr, nt = CHUNK_SHAPES[path]
    for k, bounds in enumerate(SPLITS):
        bounds = tuple(b for b in bounds if b < ni)
        chunked_vs_one_call(pm, ni, ns, nr, nt, dtype, bounds, 20 + k)


@pytest.mark.gpu
def test_chunk_accumulates_into_the_traces(pm):
    """forward with accumulate 1: y0 + A x, within one rounding per sample of y0 + (A x)"""
    import torch
    L = pm._lib
    ni, ns, nr, nt, dt = 100, 2, 3, 16, 0.004
    ts, tr = random_tables(ni, ns, nr, nt, dt, 5)
    tsd, trd = dev(ts.T), dev(tr.T)
    rng = np.random.default_rng(6)
    x, y0 = dev(rng.standard_normal(ni)), dev(rng.standard_normal(ns * nr * nt))
    ax = torch.empty_like(y0)
    assert L.lib.b2_kirchhoff(L.ctx(), x.data_ptr(), ax.data_ptr(), tsd.data_ptr(), trd.data_ptr(), ni, ns, nr, nt, dt,
                              0, L.F64, L.stream()) == 0
    y = y0.clone()
    assert c_chunk(pm, x.data_ptr(), y.data_ptr(), tsd.data_ptr(), trd.data_ptr(), ni, 0, ni, ns, nr, nt, dt, 0, 1,
                   L.F64) == 0
    ref = host(y0) + host(ax)
    mag = KREF.spread(np.abs(host(x)), ts, tr, dt, nt, np.float64).ravel() + np.abs(host(y0))
    assert np.all(np.abs(host(y) - ref) <= 2 * ni * 2.0 ** -52 * mag)


@pytest.mark.gpu
def test_chunk_error_codes_leave_y_untouched(pm):
    import torch
    L = pm._lib
    ni, ns, nr, nt = 70, 2, 3, 5
    x = torch.ones(ns * nr * nt, dtype=torch.float64, device="cuda")
    ts = torch.zeros(ns * ni, dtype=torch.float64, device="cuda")
    tr = torch.zeros(nr * ni, dtype=torch.float64, device="cuda")
    b, y = guarded(ns * nr * nt, torch.float64)
    cases = [
        (dict(x=None), ARG), (dict(y=None), ARG), (dict(ts=None), ARG), (dict(tr=None), ARG), (dict(y="x"), ARG),
        (dict(ni=0), ARG), (dict(ns=0), ARG), (dict(nr=0), ARG), (dict(nt=0), ARG),
        (dict(dt=0.0), ARG), (dict(dt=-0.004), ARG), (dict(dt=float("inf")), ARG), (dict(dt=float("nan")), ARG),
        (dict(nc=0), ARG), (dict(i0=16, nc=16), ARG), (dict(i0=1, nc=1), ARG), (dict(i0=32, nc=39), ARG),
        (dict(i0=64, nc=7), ARG), (dict(i0=96, nc=1), ARG), (dict(i0=0, nc=71), ARG),
        (dict(accumulate=2), ARG), (dict(accumulate=-1), ARG),
        (dict(dtype=L.C64), DT), (dict(dtype=L.C128), DT), (dict(dtype=L.BF16), DT), (dict(dtype=99), DT),
    ]
    for adjoint in (0, 1):
        todo = cases + ([(dict(accumulate=1), ARG)] if adjoint else [])
        for kw, want in todo:
            a = dict(x=x.data_ptr(), y=y.data_ptr(), ts=ts.data_ptr(), tr=tr.data_ptr(), ni=ni, i0=32, nc=32, ns=ns,
                     nr=nr, nt=nt, dt=0.004, accumulate=0, dtype=L.F64)
            a.update(kw)
            if a["y"] == "x":
                a["y"] = a["x"]
            rc = L.lib.b2_kirchhoff_chunk(L.ctx(), a["x"], a["y"], a["ts"], a["tr"], a["ni"], a["i0"], a["nc"], a["ns"],
                                          a["nr"], a["nt"], a["dt"], adjoint, a["accumulate"], a["dtype"], L.stream())
            assert rc == want, (kw, adjoint, rc)
        rc = L.lib.b2_kirchhoff_chunk(None, x.data_ptr(), y.data_ptr(), ts.data_ptr(), tr.data_ptr(), ni, 0, 32, ns,
                                      nr, nt, 0.004, adjoint, 0, L.F64, L.stream())
        assert rc == ARG
    torch.cuda.synchronize()
    assert torch.all(b == SENT)


@pytest.mark.gpu
def test_tables_error_codes_leave_table_untouched(pm):
    import torch
    ny, nx, nz, n = 2, 3, 4, 5
    ni = ny * nx * nz
    ay, ax, az = dev(np.arange(ny)), dev(np.arange(nx)), dev(np.arange(nz))
    pts = dev(np.zeros((3, n)))
    b, t = guarded(n * ni, torch.float64)
    cases = [dict(ax=None), dict(az=None), dict(pts=None), dict(table=None), dict(nx=0), dict(nz=0), dict(n=0),
             dict(nc=0), dict(ny=0), dict(i0=ni, nc=1), dict(i0=1, nc=ni), dict(i0=0, nc=ni + 1),
             dict(ay=None, i0=nx * nz, nc=1)]
    for kw in cases:
        a = dict(ay=ay.data_ptr(), ax=ax.data_ptr(), az=az.data_ptr(), ny=ny, nx=nx, nz=nz, pts=pts.data_ptr(), n=n,
                 i0=0, nc=ni, table=t.data_ptr())
        a.update(kw)
        rc = c_tables(pm, a["ay"], a["ax"], a["az"], a["ny"], a["nx"], a["nz"], a["pts"], a["n"], 1000.0, a["i0"],
                      a["nc"], a["table"])
        assert rc == ARG, (kw, rc)
    L = pm._lib
    assert L.lib.b2_kirchhoff_tables(None, ay.data_ptr(), ax.data_ptr(), az.data_ptr(), ny, nx, nz, pts.data_ptr(), n,
                                     1000.0, 0, ni, t.data_ptr(), L.stream()) == ARG
    torch.cuda.synchronize()
    assert torch.all(b == SENT)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the operators
# ---------------------------------------------------------------------------------------------------------------
def op_vstack(pm, P, wav, dtype="float64"):
    """the P ranks' 3-D operators of an operator case, as one MPIVStack on this GPU"""
    h, off = mgk.wavelet(wav)
    ops = []
    for r in range(P):
        z, x, t, srcs, recs, vel, y = m3.op_geometry(P, r)
        ops.append(pm.local.Kirchhoff(z, x, t, srcs, recs, vel, h, off, y=y, mode="analytic", dtype=dtype))
    return pm.MPIVStack(ops)


def bcast(pm, a):
    return pm.DistributedArray.to_dist(a, partition=pm.Partition.BROADCAST)


@pytest.fixture
def chunk_budget(pm, monkeypatch):
    """sets the table budget to ``points`` image points' tables of an operator with ns + nr points"""
    def set_budget(npts, points):
        monkeypatch.setattr(pm.local, "KIRCHHOFF_TABLE_BYTES", npts * 8 * points)
    return set_budget


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
@pytest.mark.parametrize("wav", mgk.WAVELETS)
def test_operator3d_vs_reference_fixtures(pm, P, wav):
    Op = op_vstack(pm, P, wav)
    assert not Op.ops[0].chunked and Op.ops[0].dims == (m3.OP_NY, m3.OP_NX, m3.OP_NZ)
    m, d = m3.op_inputs(P)
    y = host((Op @ bcast(pm, m)).asarray())
    ya = host((Op.H @ pm.DistributedArray.to_dist(d)).asarray())
    gy, gya = GOLD[f"{mgk.key(P, wav)}/y"], GOLD[f"{mgk.key(P, wav)}/ya"]
    np.testing.assert_allclose(y, gy, rtol=0, atol=1e-12 * np.abs(gy).max())
    if wav == "spike" and P == 1:
        np.testing.assert_array_equal(ya, gya)            # identity convolution, one rank: pylops' stacking exactly
    else:
        np.testing.assert_allclose(ya, gya, rtol=0, atol=1e-12 * np.abs(gya).max())
    Op32 = op_vstack(pm, P, wav, "float32")
    y32 = host((Op32 @ bcast(pm, m.astype(np.float32))).asarray())
    ya32 = host((Op32.H @ pm.DistributedArray.to_dist(d.astype(np.float32))).asarray())
    assert y32.dtype == np.float32 and ya32.dtype == np.float32
    np.testing.assert_allclose(y32, gy, rtol=0, atol=100 * U32 * np.abs(gy).max())
    np.testing.assert_allclose(ya32, gya, rtol=0, atol=100 * U32 * np.abs(gya).max())


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_operator3d_dottest(pm, dtype):
    Op = op_vstack(pm, 2, "ricker21", dtype)
    rng = np.random.default_rng(5)
    u = bcast(pm, rng.standard_normal(Op.shape[1]).astype(dtype))
    v = pm.DistributedArray.to_dist(rng.standard_normal(Op.shape[0]).astype(dtype))
    assert pm.dottest(Op, u, v, rtol=1e-4 if dtype == "float32" else 1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("dims", ["3d", "2d"])
def test_forced_chunks_equal_resident_bitwise(pm, chunk_budget, dims):
    """a budget lowered to 4 chunks: 64, 64, 64, 18 image points in 3-D (ni = 210), 32, 32, 32, 21 in 2-D (117)"""
    import torch
    h, off = mgk.wavelet("asym/o4")
    if dims == "3d":
        z, x, t, srcs, recs, vel, y = m3.op_geometry(1)
        points = 64
    else:
        (z, x, t, srcs, recs, vel), y = mgk.op_geometry(1), None
        points = 32
    K = pm.local.Kirchhoff
    npts = srcs.shape[1] + recs.shape[1]
    resident = {dt: K(z, x, t, srcs, recs, vel, h, off, y=y, mode="analytic", dtype=dt) for dt in ("float64", "float32")}
    chunk_budget(npts, points)
    chunked = {dt: K(z, x, t, srcs, recs, vel, h, off, y=y, mode="analytic", dtype=dt) for dt in ("float64", "float32")}
    ni = resident["float64"].ni
    assert -(-ni // points) == 4
    for dt in resident:
        assert not resident[dt].chunked and chunked[dt].chunked and chunked[dt]._nc == points
    rng = np.random.default_rng(8)
    for dt, tdt in (("float64", torch.float64), ("float32", torch.float32)):
        R, C = resident[dt], chunked[dt]
        for adjoint in (False, True):
            n = R.shape[0] if adjoint else R.shape[1]
            a = torch.as_tensor(rng.standard_normal(n)).to(tdt).cuda()
            fr, fc = (R.rmatvec, C.rmatvec) if adjoint else (R.matvec, C.matvec)
            assert torch.equal(fr(a), fc(a))
            out = torch.full((R.shape[1] if adjoint else R.shape[0],), 3.0, dtype=tdt, device="cuda")
            fc(a, out=out)
            assert torch.equal(out, fr(a))
            zc = torch.complex(a, a.flip(0)).contiguous()
            assert torch.equal(fr(zc), fc(zc))


@pytest.mark.gpu
def test_chunked_apply_allocates_nothing(pm, chunk_budget):
    import torch
    z, x, t, srcs, recs, vel, y = m3.op_geometry(1)
    chunk_budget(srcs.shape[1] + recs.shape[1], 64)
    h, off = mgk.wavelet("ricker21")
    Kop = pm.local.Kirchhoff(z, x, t, srcs, recs, vel, h, off, y=y, mode="analytic")
    assert Kop.chunked
    rng = np.random.default_rng(9)
    for adjoint in (False, True):
        nout, nin = Kop.shape[::-1] if adjoint else Kop.shape
        a = torch.as_tensor(rng.standard_normal(nin)).cuda()
        out = torch.empty(nout, dtype=torch.float64, device="cuda")
        f = Kop.rmatvec if adjoint else Kop.matvec
        f(a, out=out)
        torch.cuda.synchronize()
        before = torch.cuda.memory_stats()["allocation.all.allocated"]
        f(a, out=out)
        pm.local.apply_into(Kop.H, a, out, not adjoint)
        torch.cuda.synchronize()
        assert torch.cuda.memory_stats()["allocation.all.allocated"] - before == 0


@pytest.mark.gpu
def test_cgls_graph_replay_matches_step_loop_chunked(pm, chunk_budget):
    chunk_budget(m3.OP_NS + m3.OP_NR, 64)
    Op = op_vstack(pm, 2, "ricker21")
    assert all(op.chunked for op in Op.ops)
    rng = np.random.default_rng(12)
    y = Op @ bcast(pm, rng.standard_normal(Op.shape[1]))
    assert_cgls_replay_matches_steps(pm, Op, y, bcast(pm, np.zeros(Op.shape[1])), 25, 20)


def run_flow(pm, P):
    ops = []
    for r in range(P):
        z, x, t, srcs, recs, v0, wav, wavc, refl, y = m3.flow_setup(P, r)
        ops.append(pm.local.LSM(z, x, t, srcs, recs, v0, wav, wavc, y=y, mode="analytic").Demop)
    V = pm.MPIVStack(ops)
    d = V @ bcast(pm, refl.ravel())
    madj = V.H @ d
    minv, _, iiter, _, _, cost = pm.cgls(V, d, x0=bcast(pm, np.zeros(V.shape[1])), niter=m3.FLOW_NITER)
    return V, host(madj.asarray()), host(minv.asarray()), iiter, np.asarray(cost)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3])
def test_flow3d_vs_reference(pm, P):
    from pylops_mpi_b200.optimization.cls_basic import _graph_safe
    V, madj, minv, iiter, cost = run_flow(pm, P)
    assert _graph_safe(V)
    g = f"flow/P{P}"
    gm, gi = GOLD[f"{g}/madj"], GOLD[f"{g}/minv"]
    np.testing.assert_allclose(madj, gm, rtol=0, atol=1e-12 * np.abs(gm).max())
    assert int(iiter) == int(GOLD[f"{g}/iiter"])
    np.testing.assert_allclose(cost, GOLD[f"{g}/cost"], rtol=FLOW_COST_RTOL)
    np.testing.assert_allclose(minv, gi, rtol=0, atol=FLOW_MINV_ATOL * np.abs(gi).max())


@pytest.mark.gpu
def test_flow3d_chunked_equals_resident_bitwise(pm, chunk_budget):
    _, madj, minv, _, cost = run_flow(pm, 2)
    chunk_budget(m3.FLOW_NS + m3.FLOW_NR, 384)                    # 1188 points: chunks of 384, 384, 384, 36
    V, madj_c, minv_c, _, cost_c = run_flow(pm, 2)
    assert all(op.chunked and op._nc == 384 for op in V.ops)
    np.testing.assert_array_equal(madj_c, madj)
    np.testing.assert_array_equal(minv_c, minv)
    np.testing.assert_array_equal(cost_c, cost)


@pytest.mark.gpu
def test_operator_y_geometry_errors(pm):
    z, x, t, srcs, recs, vel, y = m3.op_geometry(1)
    K = pm.local.Kirchhoff
    with pytest.raises(NotImplementedError, match=r"y=None.*\(2, n\)"):
        K(z, x, t, srcs, recs, vel, [1.0], 0, mode="analytic")                    # 3-row geometry without y
    with pytest.raises(NotImplementedError, match=r"y=given.*\(3, n\)"):
        K(z, x, t, srcs[1:], recs[1:], vel, [1.0], 0, y=y, mode="analytic")       # 2-row geometry with y
    with pytest.raises(NotImplementedError, match="y"):
        K(z, x, t, srcs, recs[1:], vel, [1.0], 0, y=y, mode="analytic")
    lsm = pm.local.LSM(z, x, t, srcs, recs, vel, [1.0], 0, y=y, mode="analytic", dtype="float32")
    assert lsm.Demop.dims == (m3.OP_NY, m3.OP_NX, m3.OP_NZ) and lsm.Demop.dtype == np.float32


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [1, 2])
def test_multi_rank_fixtures3d(nproc):
    needs_gpus(nproc)
    run_on_ranks("test_kirchhoff3d", nproc)


def on_ranks(pm, comm):
    """each rank's MPIVStack([3-D Kirchhoff]) against its slice of the gathered fixtures, resident and in chunks,
    and the 3-D LSM flow against its fixture"""
    rank, P = comm.Get_rank(), comm.Get_size()
    BUDGET = pm.local.KIRCHHOFF_TABLE_BYTES

    def close(name, got, ref, atol_rel):
        np.testing.assert_allclose(got, ref, rtol=0, atol=atol_rel * np.abs(ref).max(), err_msg=f"[rank {rank}] {name}")

    n = m3.OP_NS * m3.OP_NR * m3.OP_NT
    ls = [(n,)] * P
    try:
        for budget in (BUDGET, (m3.OP_NS + m3.OP_NR) * 8 * 64):          # resident, then chunks of 64 image points
            pm.local.KIRCHHOFF_TABLE_BYTES = budget
            for wav in mgk.WAVELETS:
                h, off = mgk.wavelet(wav)
                z, x, t, srcs, recs, vel, y = m3.op_geometry(P, rank)
                K = pm.local.Kirchhoff(z, x, t, srcs, recs, vel, h, off, y=y, mode="analytic")
                assert K.chunked == (budget != BUDGET)
                Op = pm.MPIVStack([K])
                m, d = m3.op_inputs(P)
                yf = Op @ pm.DistributedArray.to_dist(m, partition=pm.Partition.BROADCAST)
                ya = Op.H @ pm.DistributedArray.to_dist(d, local_shapes=ls)
                k = mgk.key(P, wav)
                close(f"{k}/y", host(yf.local_array), GOLD[f"{k}/y"][rank * n:(rank + 1) * n], 1e-12)
                close(f"{k}/ya", host(ya.local_array), GOLD[f"{k}/ya"], 1e-12)
    finally:
        pm.local.KIRCHHOFF_TABLE_BYTES = BUDGET

    z, x, t, srcs, recs, v0, wav, wavc, refl, y = m3.flow_setup(P, rank)
    lsm = pm.local.LSM(z, x, t, srcs, recs, v0, wav, wavc, y=y, mode="analytic")
    VStack = pm.MPIVStack(ops=[lsm.Demop, ])
    refl_dist = pm.DistributedArray(global_shape=refl.size, partition=pm.Partition.BROADCAST)
    refl_dist[:] = refl.flatten()
    d_dist = VStack @ refl_dist
    madj = VStack.H @ d_dist
    x0 = pm.DistributedArray(VStack.shape[1], partition=pm.Partition.BROADCAST)
    x0[:] = 0
    minv, _, iiter, _, _, cost = pm.cgls(VStack, d_dist, x0=x0, niter=m3.FLOW_NITER)
    g = f"flow/P{P}"
    close(f"{g}/madj", host(madj.local_array), GOLD[f"{g}/madj"], 1e-12)
    assert int(iiter) == int(GOLD[f"{g}/iiter"])
    np.testing.assert_allclose(np.asarray(cost), GOLD[f"{g}/cost"], rtol=FLOW_COST_RTOL, err_msg=f"[rank {rank}] cost")
    close(f"{g}/minv", host(minv.local_array), GOLD[f"{g}/minv"], FLOW_MINV_ATOL)
