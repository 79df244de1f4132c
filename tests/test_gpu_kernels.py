"""GPU parity tests, kernel level: every libb200lops entry point is called through
the C ABI (ctypes) and compared with the CPU oracle / NumPy on the same seeded
inputs.  Multi-rank semantics of the stencil kernel are exercised on ONE GPU by
invoking the per-rank kernel for each simulated rank with explicit halo rows."""
import ctypes as C

import numpy as np
import pytest
import torch

import pylops_mpi_oracle as o

pytestmark = pytest.mark.gpu

KINDS = {"forward": 0, "backward": 1, "centered": 2}


@pytest.fixture(scope="module")
def L():
    import pylops_mpi_b200._lib as L
    return L


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda()


# --------------------------------------------------------------------------
# first derivative: per-rank kernel vs oracle per-rank output
# --------------------------------------------------------------------------
def run_fd_rank(L, xg, dims, P, r, kind, order, edge, h, adjoint, code):
    """apply the kernel as rank r of P on the row-block partition of xg (N x ncols)"""
    N = dims[0]
    rows = [o.local_split((N,), P, q)[0] for q in range(P)]
    off = np.cumsum([0] + rows)
    lo_need, hi_need = C.c_int(), C.c_int()
    L.check(L.lib.b2_first_derivative_halo(KINDS[kind], order, int(adjoint), C.byref(lo_need), C.byref(hi_need)))
    r0, r1 = off[r], off[r + 1]
    n_lo = min(lo_need.value, r0)
    n_hi = min(hi_need.value, N - r1)
    x = dev(xg[r0:r1])
    lo = dev(xg[r0 - n_lo:r0]) if n_lo else None
    hi = dev(xg[r1:r1 + n_hi]) if n_hi else None
    y = torch.empty_like(x)
    ncols = xg.shape[1] * (2 if np.iscomplexobj(xg) else 1)
    L.check(L.lib.b2_first_derivative(L.ctx(), x.data_ptr(), y.data_ptr(),
                                      lo.data_ptr() if lo is not None else None, n_lo,
                                      hi.data_ptr() if hi is not None else None, n_hi,
                                      r1 - r0, ncols, r0, N, KINDS[kind], order, int(edge), float(h),
                                      int(adjoint), code, L.stream()), "fd")
    return y.cpu().numpy()


@pytest.mark.parametrize("dims", [(11, 21), (600,), (100, 151), (101, 51, 10), (79, 11, 5), (64, 256), (9, 32)])
@pytest.mark.parametrize("kind,order", [("forward", 3), ("backward", 3), ("centered", 3), ("centered", 5)])
@pytest.mark.parametrize("edge", [False, True])
def test_first_derivative_per_rank_f64(L, dims, kind, order, edge):
    rng = np.random.default_rng(42)
    N, n = dims[0], int(np.prod(dims))
    for P in (1, 2, 3, 4):
        for h in (1.0, 0.4):
            for adjoint in (False, True):
                x = rng.normal(0, 10, n)
                xg = x.reshape(N, -1)
                try:
                    ref = o.first_derivative(o.to_dist(x, P), dims, h, kind, edge, order, adjoint)
                except (ValueError, IndexError):
                    D = o.first_derivative_dense(N, h, kind, edge, order)
                    full = ((D.T if adjoint else D) @ xg)
                    rows = np.cumsum([0] + [o.local_split((N,), P, q)[0] for q in range(P)])
                    ref = [full[rows[q]:rows[q + 1]].ravel() for q in range(P)]
                for r in range(P):
                    got = run_fd_rank(L, xg, dims, P, r, kind, order, edge, h, adjoint, L.F64)
                    np.testing.assert_allclose(got.ravel(), ref[r], rtol=1e-12, atol=1e-12,
                                               err_msg=f"{dims} P={P} r={r} {kind}{order} edge={edge} adj={adjoint}")


def test_first_derivative_kat_bit_exact(L):
    # plot_derivative.py:36-43 / README.md:73-94
    x = np.zeros((11, 21))
    x[5, 10] = 1.0
    y = np.concatenate([run_fd_rank(L, x, (11, 21), 2, r, "centered", 3, False, 1.0, False, L.F64) for r in range(2)])
    expect = np.zeros((11, 21))
    expect[4, 10], expect[6, 10] = 0.5, -0.5
    assert np.array_equal(y, expect)
    ref = np.concatenate(o.first_derivative(o.to_dist(x.ravel(), 2), (11, 21))).reshape(11, 21)
    assert np.array_equal(y, ref)


@pytest.mark.parametrize("kind,order", [("forward", 3), ("centered", 3), ("centered", 5)])
def test_first_derivative_f32_and_complex(L, kind, order):
    rng = np.random.default_rng(7)
    dims = (257, 96)
    x32 = rng.standard_normal(dims).astype(np.float32)
    xc = (rng.standard_normal(dims) + 1j * rng.standard_normal(dims))
    for adjoint in (False, True):
        D = o.first_derivative_dense(dims[0], 0.5, kind, True, order)
        Dm = D.T if adjoint else D
        got = np.concatenate([run_fd_rank(L, x32, dims, 3, r, kind, order, True, 0.5, adjoint, L.F32) for r in range(3)])
        np.testing.assert_allclose(got, Dm @ x32.astype(np.float64), rtol=2e-5, atol=2e-5)
        gotc = np.concatenate([run_fd_rank(L, xc, dims, 2, r, kind, order, True, 0.5, adjoint, L.F64) for r in range(2)])
        np.testing.assert_allclose(gotc, Dm @ xc, rtol=1e-12, atol=1e-12)


def test_first_derivative_missing_halo_is_an_error(L):
    x = torch.zeros((4, 32), dtype=torch.float64, device="cuda")
    y = torch.empty_like(x)
    rc = L.lib.b2_first_derivative(L.ctx(), x.data_ptr(), y.data_ptr(), None, 0, None, 0, 4, 32, 4, 12,
                                   2, 3, 0, 1.0, 0, L.F64, L.stream())
    assert rc == 2003
    with pytest.raises(L.B200Error):
        L.check(rc, "fd")


def test_first_derivative_large_properties(L):
    """full-size style checks: exact adjointness <Dx,y> = <x,D^T y> and agreement with a
    torch float32 restatement of the stencil on a > L2 array"""
    torch.manual_seed(0)
    N, ncols = 16384, 4096          # 256 MiB float32
    x = torch.randn(N, ncols, device="cuda", dtype=torch.float32)
    v = torch.randn(N, ncols, device="cuda", dtype=torch.float32)
    y = torch.empty_like(x)
    z = torch.empty_like(x)
    for kind, order in ((2, 3), (2, 5), (0, 3)):
        L.check(L.lib.b2_first_derivative(L.ctx(), x.data_ptr(), y.data_ptr(), None, 0, None, 0, N, ncols, 0, N,
                                          kind, order, 0, 1.0, 0, L.F32, L.stream()))
        L.check(L.lib.b2_first_derivative(L.ctx(), v.data_ptr(), z.data_ptr(), None, 0, None, 0, N, ncols, 0, N,
                                          kind, order, 0, 1.0, 1, L.F32, L.stream()))
        lhs = torch.dot(y.double().view(-1), v.double().view(-1)).item()
        rhs = torch.dot(x.double().view(-1), z.double().view(-1)).item()
        assert abs(lhs - rhs) <= 1e-6 * max(abs(lhs), abs(rhs), 1.0)
        ref = torch.zeros_like(x)
        if (kind, order) == (2, 3):
            ref[1:-1] = 0.5 * (x[2:] - x[:-2])
        elif (kind, order) == (2, 5):
            ref[2:-2] = x[:-4] / 12.0 - 2 * x[1:-3] / 3.0 + 2 * x[3:-1] / 3.0 - x[4:] / 12.0
        else:
            ref[:-1] = x[1:] - x[:-1]
        assert torch.allclose(y, ref, rtol=1e-5, atol=1e-5)


def test_first_derivative_host_pipeline(L):
    rng = np.random.default_rng(3)
    N, ncols = 3000, 1024
    x = rng.standard_normal((N, ncols)).astype(np.float32)
    xh = torch.as_tensor(x).pin_memory()
    yh = torch.empty_like(xh).pin_memory()
    for kind, order, adj in ((2, 3, 0), (2, 5, 1), (1, 3, 0)):
        L.check(L.lib.b2_first_derivative_host(L.ctx(), xh.data_ptr(), yh.data_ptr(), N, ncols, 0, N, kind, order, 1,
                                               2.0, adj, L.F32), "fd_host")
        name = {0: "forward", 1: "backward", 2: "centered"}[kind]
        D = o.first_derivative_dense(N, 2.0, name, True, order)
        Dm = D.T if adj else D
        # dense N x N on a column sample keeps the CPU check cheap
        cols = np.arange(0, ncols, 97)
        np.testing.assert_allclose(yh.numpy()[:, cols], Dm @ x[:, cols].astype(np.float64), rtol=2e-5, atol=2e-5)


# --------------------------------------------------------------------------
# element-wise + reductions
# --------------------------------------------------------------------------
DT = {"f32": (np.float32, 0), "f64": (np.float64, 1), "c64": (np.complex64, 2), "c128": (np.complex128, 3)}


def rnd(rng, n, npdt):
    if np.issubdtype(npdt, np.complexfloating):
        return (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(npdt)
    return rng.standard_normal(n).astype(npdt)


@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("n", [0, 1, 3, 257, 4099, 1 << 20])
def test_lincomb_mul_fill(L, dt, n):
    npdt, code = DT[dt]
    rng = np.random.default_rng(n + 1)
    x, y = rnd(rng, n, npdt), rnd(rng, n, npdt)
    xd, yd = dev(x), dev(y)
    out = torch.empty_like(xd)
    cx = np.issubdtype(npdt, np.complexfloating)
    tol = dict(rtol=2e-6, atol=2e-6) if dt in ("f32", "c64") else dict(rtol=1e-14, atol=1e-14)
    for a, b, conj in [(1.0, -1.0, 0), (2.5, 0.5, 0), (-1.0, None, 0)] + ([(1.0, None, 1), (0.5 - 2j, 1 + 1j, 0), (1j, 2.0, 1)] if cx else []):
        if n == 0:
            continue
        L.check(L.lib.b2_lincomb(L.ctx(), out.data_ptr(), L.cpair(a), xd.data_ptr(),
                                 L.cpair(b) if b is not None else None, yd.data_ptr() if b is not None else None,
                                 n, code, conj, L.stream()))
        xx = x.conj() if conj else x
        ref = a * xx + (b * y if b is not None else 0)
        np.testing.assert_allclose(out.cpu().numpy(), ref.astype(npdt), **tol)
    if n:
        L.check(L.lib.b2_mul(L.ctx(), out.data_ptr(), xd.data_ptr(), yd.data_ptr(), n, code, 0, L.stream()))
        np.testing.assert_allclose(out.cpu().numpy(), x * y, **tol)
        L.check(L.lib.b2_fill(L.ctx(), out.data_ptr(), L.cpair(3.0 - (1j if cx else 0)), n, code, L.stream()))
        assert np.all(out.cpu().numpy() == npdt(3.0 - (1j if cx else 0)))
        # unaligned views take the scalar path
        if n > 8:
            o2 = torch.empty(n + 1, dtype=xd.dtype, device="cuda")[1:]
            x2 = torch.cat([xd[:1], xd])[1:]
            L.check(L.lib.b2_lincomb(L.ctx(), o2.data_ptr(), L.cpair(2.0), x2.data_ptr(), L.cpair(1.0), yd.data_ptr(),
                                     n, code, 0, L.stream()))
            np.testing.assert_allclose(o2.cpu().numpy(), (2.0 * x + y).astype(npdt), **tol)


@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("n", [0, 1, 5, 1023, 65537, 3_000_001])
def test_dot_and_norm_partials(L, dt, n):
    npdt, code = DT[dt]
    rng = np.random.default_rng(n + 11)
    x, y = rnd(rng, n, npdt), rnd(rng, n, npdt)
    if n > 4:
        x[3] = 0
    xd, yd = dev(x), dev(y)
    out = torch.empty(2, dtype=torch.float64, device="cuda")
    x64 = x.astype(np.complex128 if np.iscomplexobj(x) else np.float64)
    y64 = y.astype(x64.dtype)
    scale = np.linalg.norm(x64) * np.linalg.norm(y64) + 1e-300
    for conj in (0, 1):
        L.check(L.lib.b2_dot(L.ctx(), xd.data_ptr() if n else None, yd.data_ptr() if n else None, n, code, conj,
                             out.data_ptr(), L.stream()))
        got = complex(*out.cpu().numpy())
        ref = np.vdot(x64, y64) if conj else np.dot(x64, y64)
        assert abs(got - ref) <= 1e-13 * scale + 1e-300
    o1 = torch.empty(1, dtype=torch.float64, device="cuda")
    a = np.abs(x64)
    refs = {0: np.count_nonzero(x), 1: a.sum(), 2: (a ** 2).sum(), 3: a.max() if n else 0.0,
            4: a.min() if n else np.inf, 5: (a ** 3).sum()}
    for kind, ref in refs.items():
        L.check(L.lib.b2_norm_partial(L.ctx(), xd.data_ptr() if n else None, n, code, kind, 3.0, o1.data_ptr(), L.stream()))
        got = o1.item()
        assert got == ref or abs(got - ref) <= 1e-12 * abs(ref), (kind, got, ref)


def test_dot_multi(L):
    rng = np.random.default_rng(5)
    n = 100_003
    for dt in ("f32", "f64", "c128"):
        npdt, code = DT[dt]
        arrs = [rnd(rng, n, npdt) for _ in range(3)]
        ds = [dev(a) for a in arrs]
        out = torch.zeros(6, dtype=torch.float64, device="cuda")
        ptrs = (C.c_void_p * 3)(*[d.data_ptr() for d in ds])
        L.check(L.lib.b2_dot_multi(L.ctx(), 3, ptrs, ptrs, n, code, 1, out.data_ptr(), L.stream()))
        res = out.cpu().numpy()
        for i, a in enumerate(arrs):
            ref = np.vdot(a.astype(np.complex128), a.astype(np.complex128)).real
            got = res[2 * i] if dt == "c128" else res[i]
            assert abs(got - ref) <= 1e-12 * ref


# --------------------------------------------------------------------------
# gemv / gemm / batched gemm
# --------------------------------------------------------------------------
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("m,n", [(1, 1), (3, 5), (101, 101), (301, 101), (64, 1000), (1000, 64), (513, 1027)])
def test_gemv_all_ops(L, dt, m, n):
    npdt, code = DT[dt]
    rng = np.random.default_rng(m * 1000 + n)
    A = rnd(rng, m * n, npdt).reshape(m, n)
    Ad = dev(A)
    A64 = A.astype(np.complex128 if np.iscomplexobj(A) else np.float64)
    tol = 2e-5 if dt in ("f32", "c64") else 1e-12
    for op, fn in ((0, lambda v: A64 @ v), (1, lambda v: A64.T @ v), (2, lambda v: A64.conj().T @ v)):
        nin, nout = (n, m) if op == 0 else (m, n)
        x = rnd(rng, nin, npdt)
        xd = dev(x)
        yd = torch.empty(nout, dtype=xd.dtype, device="cuda")
        L.check(L.lib.b2_gemv(L.ctx(), Ad.data_ptr(), n, m, n, xd.data_ptr(), yd.data_ptr(), op, code, code, L.stream()))
        ref = fn(x.astype(A64.dtype))
        scale = np.abs(A64).sum(axis=1 if op == 0 else 0).max() * np.abs(x).max() + 1e-30
        np.testing.assert_allclose(yd.cpu().numpy(), ref, rtol=tol, atol=tol * scale)


@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("m", [1, 3, 4, 9, 130])
def test_gemv_long_rows_split_kernel(L, dt, m):
    """rows of >= 32 KB take the row-splitting kernel (8 warps sweep 4 rows together): ragged row counts, a row
    pitch larger than n (view of a wider matrix, scalar remainder columns) and every element type vs float64"""
    npdt, code = DT[dt]
    esz = np.dtype(npdt).itemsize
    vecw = 16 // esz
    n = 32768 // esz + 3 * 256 * vecw + 5 * vecw + (1 if vecw > 1 else 0)   # >= 32 KB, ragged in every loop of the kernel
    lda = -(-n // vecw) * vecw + 2 * vecw                                    # pitch: multiple of 16 bytes, > n
    rng = np.random.default_rng(m * 31 + esz)
    A = rnd(rng, m * lda, npdt).reshape(m, lda)
    x = rnd(rng, n, npdt)
    Ad, xd = dev(A), dev(x)
    yd = torch.empty(m, dtype=xd.dtype, device="cuda")
    L.check(L.lib.b2_gemv(L.ctx(), Ad.data_ptr(), lda, m, n, xd.data_ptr(), yd.data_ptr(), 0, code, code, L.stream()))
    A64 = A[:, :n].astype(np.complex128 if np.iscomplexobj(A) else np.float64)
    ref = A64 @ x.astype(A64.dtype)
    tol = 2e-5 if dt in ("f32", "c64") else 1e-12
    scale = np.abs(A64).sum(axis=1).max() * np.abs(x).max() + 1e-30
    np.testing.assert_allclose(yd.cpu().numpy(), ref, rtol=tol, atol=tol * scale)


def test_gemv_bf16_long_rows(L):
    torch.manual_seed(2)
    for m, n in ((5, 32768), (64, 16384 + 8 * 300)):
        A = (torch.randn(m, n, device="cuda") / 180).to(torch.bfloat16)
        x = torch.randn(n, device="cuda")
        y = torch.empty(m, device="cuda")
        L.check(L.lib.b2_gemv(L.ctx(), A.data_ptr(), n, m, n, x.data_ptr(), y.data_ptr(), 0, L.BF16, L.F32, L.stream()))
        ref = A.double() @ x.double()
        assert torch.allclose(y.double(), ref, rtol=1e-4, atol=1e-4)


def test_gemv_bf16(L):
    torch.manual_seed(1)
    m, n = 1024, 2048
    A = (torch.randn(m, n, device="cuda") / 45).to(torch.bfloat16)
    for op in (0, 1):
        x = torch.randn(n if op == 0 else m, device="cuda")
        y = torch.empty(m if op == 0 else n, device="cuda")
        L.check(L.lib.b2_gemv(L.ctx(), A.data_ptr(), n, m, n, x.data_ptr(), y.data_ptr(), op, L.BF16, L.F32, L.stream()))
        A64 = A.double()
        ref = (A64 @ x.double()) if op == 0 else (A64.T @ x.double())
        assert torch.allclose(y.double(), ref, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("m,n,k", [(64, 64, 64), (37, 37, 37), (50, 40, 30), (3, 5, 4), (1, 1, 2), (2, 3, 1), (130, 70, 33)])
def test_gemm_simt(L, dt, m, n, k):
    npdt, code = DT[dt]
    rng = np.random.default_rng(m + 7 * n + 13 * k)
    tol = 3e-5 if dt in ("f32", "c64") else 1e-12
    B = rnd(rng, k * n, npdt).reshape(k, n)
    for op in (0, 1, 2):
        A = rnd(rng, m * k, npdt).reshape((m, k) if op == 0 else (k, m))
        A64 = A.astype(np.complex128 if np.iscomplexobj(A) else np.float64)
        opA = A64 if op == 0 else (A64.T if op == 1 else A64.conj().T)
        Ad, Bd = dev(A), dev(B)
        Cd = torch.ones((m, n), dtype=Ad.dtype, device="cuda")
        L.check(L.lib.b2_gemm(L.ctx(), Ad.data_ptr(), A.shape[1], Bd.data_ptr(), n, Cd.data_ptr(), n, m, n, k, op, 0,
                              code, L.stream()))
        ref = opA @ B.astype(A64.dtype)
        scale = np.abs(ref).max() + 1
        np.testing.assert_allclose(Cd.cpu().numpy(), ref, rtol=tol, atol=tol * scale)
        L.check(L.lib.b2_gemm(L.ctx(), Ad.data_ptr(), A.shape[1], Bd.data_ptr(), n, Cd.data_ptr(), n, m, n, k, op, 1,
                              code, L.stream()))
        np.testing.assert_allclose(Cd.cpu().numpy(), 2 * ref, rtol=tol, atol=2 * tol * scale)


@pytest.mark.parametrize("nz", [5, 1])
@pytest.mark.parametrize("dt", ["f32", "c64", "f64", "c128"])
def test_batched_gemm_fredholm_kat(L, nz, dt):
    # test_fredholm.py:36-95: G = arange(21*4*6) (- 1j * same), x = ones (+ 1j)
    npdt, code = DT[dt]
    cx = np.issubdtype(npdt, np.complexfloating)
    nsl, nx, ny = 21, 4, 6
    G = np.arange(nsl * nx * ny, dtype=np.float64).reshape(nsl, nx, ny)
    G = (G - 1j * G) if cx else G
    x = np.ones((nsl, ny, nz)) + (1j if cx else 0)
    Gd, xd = dev(G.astype(npdt)), dev(x.astype(npdt))
    yd = torch.empty((nsl, nx, nz), dtype=Gd.dtype, device="cuda")
    L.check(L.lib.b2_batched_gemm(L.ctx(), Gd.data_ptr(), xd.data_ptr(), yd.data_ptr(), nsl, nx, ny, nz, 0, code, L.stream()))
    ref = np.matmul(G, x)
    tol = 1e-5 if dt in ("f32", "c64") else 1e-13
    np.testing.assert_allclose(yd.cpu().numpy(), ref, rtol=tol)
    xa = torch.empty((nsl, ny, nz), dtype=Gd.dtype, device="cuda")
    L.check(L.lib.b2_batched_gemm(L.ctx(), Gd.data_ptr(), yd.data_ptr(), xa.data_ptr(), nsl, nx, ny, nz, 1, code, L.stream()))
    refa = np.matmul(G.conj().transpose(0, 2, 1), yd.cpu().numpy().astype(G.dtype))
    np.testing.assert_allclose(xa.cpu().numpy(), refa, rtol=tol * 10)


# --------------------------------------------------------------------------
# bf16 tile product on the tensor cores (wgmma)
# --------------------------------------------------------------------------
# Operands and outputs of the tensor-core tests live inside larger buffers: every element outside the view holds a
# sentinel bit pattern (a NaN payload), so a load past a row end shows up in the result and a stray store shows up as
# a changed guard element, without leaving the allocation.
SENT32, SENT16 = 0x7FC0DEAD, 0x7FAD
_INT_VIEW = {torch.float32: torch.int32, torch.bfloat16: torch.int16}


def guarded(rows, cols, ld, off, dtype=torch.float32, sentinel=None):
    """(buffer, view): a rows x cols view with row pitch ld at element offset off of a buffer filled with sentinel"""
    buf = torch.empty(off + rows * ld + ld, dtype=dtype, device="cuda")
    buf.view(_INT_VIEW[dtype]).fill_(sentinel if sentinel is not None else (SENT32 if dtype == torch.float32 else SENT16))
    return buf, buf.as_strided((rows, cols), (ld, 1), off)


def guards_intact(buf, view, sentinel=None):
    mask = torch.ones(buf.numel(), dtype=torch.bool, device=buf.device)
    mask.as_strided(view.shape, view.stride(), view.storage_offset()).fill_(False)
    sentinel = sentinel if sentinel is not None else (SENT32 if buf.dtype == torch.float32 else SENT16)
    return bool((buf.view(_INT_VIEW[buf.dtype])[mask] == sentinel).all())


def bits(t):
    return t.contiguous().view(_INT_VIEW[t.dtype])


def pitched_bf16(rows, cols, gen, scale=1 / 8):
    """bf16 rows x cols view one row into a buffer with row pitch > cols (a multiple of 8, as TMA needs); every
    element outside the view is 1e4, so reading it would wreck the product"""
    ld = -(-cols // 8) * 8 + 8
    buf = torch.full(((rows + 2) * ld,), 1e4, dtype=torch.bfloat16, device="cuda")
    view = buf.as_strided((rows, cols), (ld, 1), ld)
    view.copy_((torch.randn(rows, cols, device="cuda", generator=gen) * scale).to(torch.bfloat16))
    return buf, view, ld


def sm_count(L):
    n = C.c_int()
    L.check(L.lib.b2_ctx_sm_count(L.ctx(), C.byref(n)))
    return n.value


def gemm_c_layout(m, n, layout):
    """C as a guarded interior view: "vec" = 8-byte aligned base and even ldc (paired stores), "odd" = base one float
    off and odd ldc (scalar stores)"""
    co = 2 if layout == "vec" else 1
    ldc = n + co + 2
    if ldc % 2 != (0 if layout == "vec" else 1):
        ldc += 1
    return guarded(m, n, ldc, 2 * ldc + co)


# 128 x 256 tiles: more tiles than SMs, so CTAs move on to further tiles (ring stage / phase carried across tiles,
# accumulator reset, grouped rasterisation with a partial last group of row tiles)
GEMM_MULTI_TILE = [(2176, 2304, 200), (4104, 2056, 72), (4096, 4096, 8)]


@pytest.mark.parametrize("m,n,k", [(128, 256, 64), (128, 256, 256), (256, 512, 128), (1024, 1024, 1024),
                                   (200, 264, 72), (8, 8, 8), (136, 40, 1000), (8, 16, 24), (384, 256, 64),
                                   (130, 77, 40)] + GEMM_MULTI_TILE + [(256, 512, 16424)])
@pytest.mark.parametrize("op", [0, 1, 2])
def test_gemm_bf16_wgmma(L, m, n, k, op):
    """every C layout, paired (vector) and scalar stores, gives the same bits within the bound, nothing outside C"""
    if (m, n, k) in GEMM_MULTI_TILE:
        assert -(-m // 128) * -(-n // 256) > sm_count(L)
    gen = torch.Generator(device="cuda").manual_seed(m * 7 + n * 3 + k + op)
    Abuf, A, lda = pitched_bf16(m, k, gen) if op == 0 else pitched_bf16(k, m, gen)
    Bbuf, B, ldb = pitched_bf16(k, n, gen)
    A64 = A.double() if op == 0 else A.double().T
    ref = A64 @ B.double()
    # fp32 accumulation of exact bf16 products: error <= ~k * eps32 * sum|a||b|
    bound = (A64.abs() @ B.double().abs()) * (k * 6e-8) + 1e-6
    results = []
    for layout in ("vec", "odd"):
        Cbuf, Cm = gemm_c_layout(m, n, layout)
        Cm.fill_(7.0)
        ldc = Cm.stride(0)
        L.check(L.lib.b2_gemm_bf16(L.ctx(), A.data_ptr(), lda, B.data_ptr(), ldb, Cm.data_ptr(), ldc, m, n, k, op, 0,
                                   L.stream()), "b2_gemm_bf16")
        torch.cuda.synchronize()
        err = (Cm.double() - ref).abs()
        assert bool((err <= bound).all()), f"max err {err.max().item()} at {m},{n},{k},{op} {layout}"
        assert guards_intact(Cbuf, Cm), f"store outside C ({layout})"
        results.append(bits(Cm))
        if op == 2:   # real bf16: H is T, bit for bit
            Ct = torch.empty(m, n, device="cuda")
            L.check(L.lib.b2_gemm_bf16(L.ctx(), A.data_ptr(), lda, B.data_ptr(), ldb, Ct.data_ptr(), n, m, n, k, 1, 0,
                                       L.stream()), "b2_gemm_bf16")
            assert torch.equal(bits(Ct), bits(Cm))
        # accumulate into C
        L.check(L.lib.b2_gemm_bf16(L.ctx(), A.data_ptr(), lda, B.data_ptr(), ldb, Cm.data_ptr(), ldc, m, n, k, op, 1,
                                   L.stream()), "b2_gemm_bf16")
        err = (Cm.double() - 2 * ref).abs()
        assert bool((err <= 2 * bound + 1e-5).all()), f"accumulate, {layout}"
        assert guards_intact(Cbuf, Cm), f"store outside C (accumulate, {layout})"
    assert torch.equal(results[0], results[1]), "scalar stores differ from paired stores"


@pytest.mark.parametrize("layout", ["vec", "odd"])
def test_gemm_bf16_k0(L, layout):
    """k = 0: the product is empty, so C is zeroed (accumulate 0) or left as it is (accumulate 1)"""
    m, n = 300, 270
    A = torch.zeros(8, device="cuda", dtype=torch.bfloat16)
    Cbuf, Cm = gemm_c_layout(m, n, layout)
    Cm.copy_(torch.randn(m, n, device="cuda"))
    before = Cm.clone()
    L.check(L.lib.b2_gemm_bf16(L.ctx(), A.data_ptr(), 8, A.data_ptr(), 8, Cm.data_ptr(), Cm.stride(0), m, n, 0, 0, 1,
                               L.stream()), "b2_gemm_bf16")
    assert torch.equal(bits(Cm), bits(before)) and guards_intact(Cbuf, Cm)
    L.check(L.lib.b2_gemm_bf16(L.ctx(), A.data_ptr(), 8, A.data_ptr(), 8, Cm.data_ptr(), Cm.stride(0), m, n, 0, 0, 0,
                               L.stream()), "b2_gemm_bf16")
    assert torch.equal(bits(Cm), torch.zeros(m, n, dtype=torch.int32, device="cuda")) and guards_intact(Cbuf, Cm)


def ptr_array(ptrs):
    return (C.c_void_p * len(ptrs))(*ptrs)


@pytest.mark.parametrize("nseg", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("seg_cols", [32, 96, 160, 288])
def test_gemm_bf16_seg(L, nseg, seg_cols):
    """column-segmented epilogue: segment c of the output goes to its own buffer; the 256-column tiles straddle
    segment boundaries.  Same kernel as b2_gemm_bf16 with only the store address changed, so every segment must
    equal the matching columns of the plain product bit for bit."""
    m, k, n = 1000, 200, nseg * seg_cols          # 8 row tiles, the last one ragged; 4 k-blocks, the last one ragged
    for op in (0, 1):
        gen = torch.Generator(device="cuda").manual_seed(nseg * 1000 + seg_cols + op)
        _, A, lda = pitched_bf16(m, k, gen) if op == 0 else pitched_bf16(k, m, gen)
        _, B, ldb = pitched_bf16(k, n, gen)
        plain = torch.empty(m, n, device="cuda")
        L.check(L.lib.b2_gemm_bf16(L.ctx(), A.data_ptr(), lda, B.data_ptr(), ldb, plain.data_ptr(), n, m, n, k, op, 0,
                                   L.stream()), "b2_gemm_bf16")
        ldc = seg_cols + 8
        segs = [guarded(m, seg_cols, ldc, ldc + 4) for _ in range(nseg)]
        L.check(L.lib.b2_gemm_bf16_seg(L.ctx(), A.data_ptr(), lda, B.data_ptr(), ldb,
                                       ptr_array([v.data_ptr() for _, v in segs]), nseg, seg_cols, ldc, m, n, k, op,
                                       L.stream()), "b2_gemm_bf16_seg")
        for c, (buf, v) in enumerate(segs):
            assert torch.equal(bits(v), bits(plain[:, c * seg_cols:(c + 1) * seg_cols])), f"segment {c} op {op}"
            assert guards_intact(buf, v), f"store outside segment {c} op {op}"


def test_gemm_bf16_seg_argument_errors(L):
    m, k = 64, 64
    A = torch.zeros(m * k, device="cuda", dtype=torch.bfloat16)
    segs = [torch.zeros(m * 400, device="cuda") for _ in range(9)]
    arr = ptr_array([s.data_ptr() for s in segs])

    def call(nseg, seg_cols, n, ldc=400, ptrs=arr):
        return L.lib.b2_gemm_bf16_seg(L.ctx(), A.data_ptr(), k, A.data_ptr(), 8, ptrs, nseg, seg_cols, ldc, m, n, k, 0,
                                      L.stream())
    assert call(2, 48, 96) == 2002            # seg_cols % 32
    assert call(2, 32, 96) == 2002            # n != nseg * seg_cols
    assert call(0, 32, 32) == 2002
    assert call(9, 32, 288) == 2002
    assert call(2, 32, 64, ldc=402) == 2002   # ldc % 4
    bad = ptr_array([segs[0].data_ptr(), segs[1].data_ptr() + 4])
    assert call(2, 32, 64, ptrs=bad) == 2006  # misaligned segment base
    torch.cuda.synchronize()


# fp32 -> bf16 edge cases: round-to-nearest-even ties and near-ties, +-0, fp32 subnormals (incl. ties), the largest
# float (rounds to inf), +-inf, NaNs
_CAST_SPECIALS = np.array([0x00000000, 0x80000000, 0x00000001, 0x00008000, 0x00018000, 0x80008000, 0x007FFFFF,
                           0x807FFFFF, 0x00400000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7F800001,
                           0x7F7FFFFF, 0x7F7F8000, 0x7F7E8000, 0x3F808000, 0x3F818000, 0xBF818000, 0x3F807FFF,
                           0x3F808001], dtype=np.uint32)


@pytest.mark.parametrize("rows,cols,ld_src,ld_dst,dst_off", [
    (37, 64, 64, 72, 0),        # vector path
    (37, 64, 68, 80, 0),        # vector path, pitched source
    (4096, 2048, 2056, 2056, 0),  # vector path, grid-stride loop
    (37, 61, 61, 64, 0),        # scalar: cols % 8
    (37, 64, 67, 72, 0),        # scalar: source pitch not a multiple of 4
    (37, 64, 64, 72, 1),        # scalar: destination not 16-byte aligned
    (1500, 1001, 1003, 1010, 0),  # scalar, grid-stride loop
])
@pytest.mark.parametrize("ndst", [1, 2, 5, 8])
def test_cast_bf16_multi(L, rows, cols, ld_src, ld_dst, dst_off, ndst):
    rng = np.random.default_rng(rows + cols + ld_src + ndst)
    src = (rng.standard_normal((rows, ld_src)) * 2.0 ** rng.integers(-30, 30, (rows, ld_src))).astype(np.float32)
    sb = src.view(np.uint32)
    sel = rng.random(sb.shape) < 0.25                                 # exact ties between two bf16 values
    sb[sel] = (sb[sel] & 0xFFFF0000) | 0x8000
    sel = rng.random(sb.shape) < 0.1                                  # one ulp either side of a tie
    sb[sel] = (sb[sel] & 0xFFFF0000) | rng.choice([0x7FFF, 0x8001], size=int(sel.sum())).astype(np.uint32)
    pos = rng.choice(rows * cols, size=min(rows * cols, 4 * len(_CAST_SPECIALS)), replace=False)
    sb[pos // cols, pos % cols] = np.resize(_CAST_SPECIALS, len(pos))
    src_d = dev(src)
    dsts = [guarded(rows, cols, ld_dst, ld_dst + dst_off, torch.bfloat16) for _ in range(ndst)]
    L.check(L.lib.b2_cast_bf16_multi(L.ctx(), src_d.data_ptr(), ld_src, rows, cols,
                                     ptr_array([v.data_ptr() for _, v in dsts]), ndst, ld_dst, L.stream()),
            "b2_cast_bf16_multi")
    # round to nearest even on the bit pattern (no flush of subnormals); torch's own cast must agree
    u = np.ascontiguousarray(sb[:, :cols]).astype(np.uint64)
    ref = torch.as_tensor(((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16).view(np.int16))
    ref_nan = torch.as_tensor(np.isnan(src[:, :cols]))
    assert torch.equal(bits(src_d[:, :cols].to(torch.bfloat16).cpu())[~ref_nan], ref[~ref_nan])
    for d, (buf, v) in enumerate(dsts):
        got = v.cpu()
        assert torch.equal(torch.isnan(got), ref_nan), f"destination {d}: NaN pattern"
        assert torch.equal(bits(got)[~ref_nan], ref[~ref_nan]), f"destination {d}"
        assert guards_intact(buf, v), f"store outside destination {d}"


@pytest.mark.parametrize("rows,cols,ld_in,out_off", [
    (33, 64, 68, 0),            # vector path, pitched slots
    (1200, 2048, 2052, 0),      # vector path, grid-stride loop
    (33, 61, 64, 0),            # scalar: cols % 4
    (33, 64, 67, 0),            # scalar: odd slot pitch
    (33, 64, 64, 1),            # scalar: output not 16-byte aligned
])
def test_sum_slots(L, rows, cols, ld_in, out_off):
    """out = slot 0 + slot 1 + ... in slot order, bit for bit against a float32 sum taken one slot at a time"""
    rng = np.random.default_rng(rows * cols + ld_in + out_off)
    slot_stride = (rows + 1) * ld_in
    for nslots in range(1, 9):
        slots = np.full(nslots * slot_stride, np.nan, dtype=np.float32)   # padding: NaN, read by nobody
        vals = (rng.standard_normal((nslots, rows, cols)) * 2.0 ** rng.integers(-12, 12, (nslots, rows, cols)))
        vals = vals.astype(np.float32)
        for s in range(nslots):
            slots[s * slot_stride:s * slot_stride + rows * ld_in].reshape(rows, ld_in)[:, :cols] = vals[s]
        ref = vals[0].copy()
        for s in range(1, nslots):
            ref = ref + vals[s]
        slots_d = dev(slots)
        buf, out = guarded(1, rows * cols, rows * cols, 4 + out_off)
        L.check(L.lib.b2_sum_slots(L.ctx(), slots_d.data_ptr(), slot_stride, nslots, ld_in, out.data_ptr(), rows, cols,
                                   L.stream()), "b2_sum_slots")
        got = out.cpu().numpy().reshape(rows, cols)
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), f"nslots {nslots}"
        assert guards_intact(buf, out), f"store outside out, nslots {nslots}"


def test_gemm_bf16_alignment_error_is_loud(L):
    A = torch.zeros(8, 12, device="cuda", dtype=torch.bfloat16)
    B = torch.zeros(12, 8, device="cuda", dtype=torch.bfloat16)
    Cm = torch.zeros(8, 8, device="cuda")
    rc = L.lib.b2_gemm_bf16(L.ctx(), A.data_ptr(), 12, B.data_ptr(), 8, Cm.data_ptr(), 8, 8, 8, 12, 0, 0, L.stream())
    assert rc == 2006


def test_gemm_bf16_worker_shapes():
    """the tensor-core kernel on multi-tile shapes (several 128-row tiles, ragged m / n / k) and an 8192^3 timing,
    in a process of its own (first use of the kernel: function attributes, tensor-map encoder)"""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, os.path.join(here, "gemm_worker.py")], capture_output=True, text=True,
                       timeout=240)
    assert r.returncode == 0 and "GEMM_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


# --------------------------------------------------------------------------
# MPIFredholm1 split-precision product on the tensor cores (b2_fredholm_plan_* / b2_fredholm_apply)
# --------------------------------------------------------------------------
# Componentwise, scale-invariant bound |y - y_ref| <= gamma (|op(G)| |x|), gamma = (c_split + K'/8) 2^-24, K' = real
# contraction length (2K for complex).  c_split from the operand format (fredholm_tc.cu): fp16x2 keeps 22 bits per
# operand and drops lo*lo, 3 * 2^-22 per product, c_split = 16.  K'/8 allows 2u per fp32 tensor-core accumulation over
# a k16 step.
C_SPLIT = 16


class FredholmPlan:
    """b2_fredholm_plan for G (torch, nsl x nx x ny, float32 or complex64)"""

    def __init__(self, L, G, nz):
        self.L, self.G, self.nz = L, G, nz
        self.h = C.c_void_p()
        nsl, nx, ny = G.shape
        L.check(L.lib.b2_fredholm_plan_create(L.ctx(), G.data_ptr(), nsl, nx, ny, nz, L.code(G.dtype),
                                              C.byref(self.h)), "b2_fredholm_plan_create")

    def apply(self, x, adjoint, y=None, peers=()):
        nsl, nx, ny = self.G.shape
        if y is None:
            y = torch.empty((nsl, ny if adjoint else nx, self.nz), dtype=self.G.dtype, device="cuda")
        self.L.check(self.L.lib.b2_fredholm_apply(self.h, x.data_ptr(), y.data_ptr(),
                                                  ptr_array([p.data_ptr() for p in peers]) if peers else None,
                                                  len(peers), int(adjoint), self.L.stream()), "b2_fredholm_apply")
        return y

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.L.lib.b2_fredholm_plan_destroy(self.h)


def fredholm_check(G, x, y, adjoint, what=""):
    """y against op(G) x in float64 / complex128, componentwise bound above"""
    cx = G.is_complex()
    wide = torch.complex128 if cx else torch.float64
    opG = G.to(wide)
    opG = opG.conj().transpose(1, 2) if adjoint else opG
    ref = opG @ x.to(wide)
    if cx:
        M = (opG.real.abs() + opG.imag.abs()) @ (x.real.double().abs() + x.imag.double().abs())
    else:
        M = opG.abs() @ x.double().abs()
    kp = opG.shape[2] * (2 if cx else 1)
    bound = (C_SPLIT + kp / 8) * 2.0 ** -24 * M
    d = y.to(wide) - ref
    parts = (d.real, d.imag) if cx else (d,)
    for p in parts:
        ok = p.abs() <= bound
        if not bool(ok.all()):
            i = torch.nonzero(~ok)[0].tolist()
            raise AssertionError(f"{what}: {int((~ok).sum())} entries outside the bound, first {i}: "
                                 f"y {y[tuple(i)].item()} ref {ref[tuple(i)].item()} bound {bound[tuple(i)].item()}")


def sign_unit(rng, shape, cx):
    """random signs, magnitudes in [1, 2): every scale applied afterwards is the only source of dynamic range"""
    def one():
        return rng.choice([-1.0, 1.0], size=shape) * rng.uniform(1.0, 2.0, size=shape)
    return one() + 1j * one() if cx else one()


def to_dev(a, cx):
    return torch.as_tensor(a.astype(np.complex64 if cx else np.float32)).cuda()


def distinct_pow2(rng, n, lo=-30, hi=30):
    """n exponents in [lo, hi]; any 8 consecutive ones are distinct"""
    return np.resize(rng.permutation(np.arange(lo, hi + 1)), n)


@pytest.mark.parametrize("cx", [False, True])
@pytest.mark.parametrize("adjoint", [False, True])
def test_fredholm_tc_scaled_inputs(L, cx, adjoint):
    """rows of op(G) and columns of x scaled by distinct powers 2^[-30, 30], entries down to 2^-24 below their
    column's maximum, one all-zero row of op(G) and one all-zero column of x (exact zeros in y).  fp16x2 scales every
    row of op(G) and every column of x separately and undoes the scales in the epilogue: an off-by-one in either
    shows up here."""
    rng = np.random.default_rng(100 + 4 * cx + 2 * adjoint)
    nsl, nx, ny, nz = 3, 70, 90, 40
    m, K = (ny, nx) if adjoint else (nx, ny)
    G = sign_unit(rng, (nsl, nx, ny), cx)
    er = 2.0 ** distinct_pow2(rng, m)
    zr = 13
    if adjoint:          # rows of G^H = columns of G
        G *= er[None, None, :]
        G[:, :, zr] = 0
    else:
        G *= er[None, :, None]
        G[:, zr, :] = 0
    x = sign_unit(rng, (nsl, K, nz), cx) * 2.0 ** -rng.integers(0, 24, (nsl, K, nz))
    x *= 2.0 ** distinct_pow2(rng, nz)[None, None, :]
    zc = 7
    x[:, :, zc] = 0
    Gd, xd = to_dev(G, cx), to_dev(x, cx)
    with FredholmPlan(L, Gd, nz) as pl:
        y = pl.apply(xd, adjoint)
        fredholm_check(Gd, xd, y, adjoint, "scaled")
        assert bool((y[:, zr, :] == 0).all()) and bool((y[:, :, zc] == 0).all())


@pytest.mark.parametrize("eg,ex", [(-118, 118), (118, -118), (-62, -62)])
@pytest.mark.parametrize("cx", [False, True])
@pytest.mark.parametrize("adjoint", [False, True])
def test_fredholm_tc_extreme_magnitudes(L, eg, ex, cx, adjoint):
    """G scaled by 2^eg and x by 2^ex.  For (-118, 118) and the reverse the products are O(1): the fp16x2 scales must
    reach 2^+-126 for the scaled operands to stay finite fp16.  For (-62, -62) the result is a normal float32
    (~2^-120) although the product of the two inverse scales is below the float32 range."""
    rng = np.random.default_rng(1000 + eg + 3 * ex + 2 * cx + adjoint)
    nsl, nx, ny, nz = 2, 40, 56, 24
    G = sign_unit(rng, (nsl, nx, ny), cx) * 2.0 ** eg
    x = sign_unit(rng, (nsl, nx if adjoint else ny, nz), cx) * 2.0 ** ex
    Gd, xd = to_dev(G, cx), to_dev(x, cx)
    with FredholmPlan(L, Gd, nz) as pl:
        y = pl.apply(xd, adjoint)
        assert bool(torch.isfinite(torch.view_as_real(y) if cx else y).all()), "non-finite y for finite inputs"
        fredholm_check(Gd, xd, y, adjoint, f"G*2^{eg}, x*2^{ex}")


@pytest.mark.parametrize("e", [-62, 80])
@pytest.mark.parametrize("cx", [False, True])
@pytest.mark.parametrize("adjoint", [False, True])
def test_fredholm_tc_h2_exact_cancellation(L, e, cx, adjoint):
    """fp16x2 with G and x both scaled by 2^e and products that cancel exactly: y must be exactly zero.  The inverse
    scales of a row of op(G) and a column of x then multiply to a power of two outside the float32 range (2^-152,
    2^132), which must not turn the zero into 0 * inf = NaN."""
    rng = np.random.default_rng(800 + e + 2 * cx + adjoint)
    nsl, nx, ny, nz = 2, 48, 40, 16
    K = nx if adjoint else ny
    # 11-bit values: every split is exact (lo planes zero), so every partial sum is exact and the pairs cancel
    G = np.ones((nsl, nx, ny)) * (1 + 1j if cx else 1) * 2.0 ** e
    sign = np.where(np.arange(K) % 2 == 0, 1.0, -1.0)[None, :, None]
    u = 1 + rng.integers(0, 1024, (nsl, K // 2, nz)) / 1024
    x = sign * np.repeat(u, 2, axis=1) * (1 - 1j if cx else 1) * 2.0 ** e
    Gd, xd = to_dev(G, cx), to_dev(x, cx)
    with FredholmPlan(L, Gd, nz) as pl:
        y = pl.apply(xd, adjoint)
        assert bool((y == 0).all()), f"{int((y != 0).sum())} nonzero entries, e.g. {y.flatten()[torch.nonzero((y != 0).flatten())[0]].item()}"


@pytest.mark.parametrize("cx,shape", [(True, (160, 200, 136, 40)), (False, (50, 130, 260, 300))])
def test_fredholm_tc_multi_tile(L, cx, shape):
    """more than two 128 x 128 output tiles per SM in both directions: CTAs move through several tiles and slices
    (ring stage / phase across tiles, accumulator reset).  The real shape packs x with the generic kernel forward
    (K = 260 > 256) and with the single-pass one in the adjoint."""
    nsl, nx, ny, nz = shape
    n = nz * (2 if cx else 1)
    for m in (nx, ny):
        assert nsl * -(-m // 128) * -(-n // 128) > 2 * sm_count(L)
    rng = np.random.default_rng(300 + nx)
    Gd = to_dev(sign_unit(rng, (nsl, nx, ny), cx), cx)
    with FredholmPlan(L, Gd, nz) as pl:
        for adjoint in (False, True):
            xd = to_dev(sign_unit(rng, (nsl, nx if adjoint else ny, nz), cx), cx)
            fredholm_check(Gd, xd, pl.apply(xd, adjoint), adjoint, f"adjoint={adjoint}")


@pytest.mark.parametrize("cx", [False, True])
@pytest.mark.parametrize("nz", [1, 17, 33])
def test_fredholm_tc_pack_kernels_agree(L, cx, nz):
    """a contraction over K <= 256 values of k packs x with the single-pass kernel.  The same product with the
    contraction padded by zeros to K = 257 (zero columns of G and zero rows of x forward, zero rows of G and x in the
    adjoint) packs x with the generic kernel.  The padding leaves every row and column scale unchanged and adds only
    zero products, so both kernels must build identical planes and scales, hence bit-identical y"""
    rng = np.random.default_rng(400 + nz + 2 * cx)
    nsl, nx, ny, kpadded = 2, 100, 200, 257
    G = sign_unit(rng, (nsl, nx, ny), cx) * 2.0 ** rng.integers(-8, 8, (nsl, nx, 1))
    Gd = to_dev(G, cx)
    for adjoint in (False, True):
        x = sign_unit(rng, (nsl, nx if adjoint else ny, nz), cx) * 2.0 ** rng.integers(-20, 20, (1, 1, nz))
        xd = to_dev(x, cx)
        pad = kpadded - x.shape[1]
        Gp = np.pad(G, ((0, 0), (0, pad), (0, 0)) if adjoint else ((0, 0), (0, 0), (0, pad)))
        xp = np.pad(x, ((0, 0), (0, pad), (0, 0)))
        ys = []
        for g, xx in ((Gd, xd), (to_dev(Gp, cx), to_dev(xp, cx))):
            with FredholmPlan(L, g, nz) as pl:
                ys.append(pl.apply(xx, adjoint))
        fredholm_check(Gd, xd, ys[0], adjoint, "single-pass pack")
        assert torch.equal(bits(torch.view_as_real(ys[0]) if cx else ys[0]),
                           bits(torch.view_as_real(ys[1]) if cx else ys[1])), f"adjoint={adjoint}"


@pytest.mark.parametrize("cx", [False, True])
def test_fredholm_tc_repeated_applies(L, cx):
    """one plan, several applies: forward x1, forward x2 (other column scales), adjoint, forward x1 again, which must
    reproduce the first result bit for bit (no stale scales or planes from the applies in between)"""
    rng = np.random.default_rng(500 + 2 * cx)
    nsl, nx, ny, nz = 3, 96, 80, 24
    Gd = to_dev(sign_unit(rng, (nsl, nx, ny), cx), cx)
    x1 = to_dev(sign_unit(rng, (nsl, ny, nz), cx) * 2.0 ** distinct_pow2(rng, nz)[None, None, :], cx)
    x2 = to_dev(sign_unit(rng, (nsl, ny, nz), cx) * 2.0 ** distinct_pow2(rng, nz)[None, None, :], cx)
    x3 = to_dev(sign_unit(rng, (nsl, nx, nz), cx) * 2.0 ** distinct_pow2(rng, nz)[None, None, :], cx)
    with FredholmPlan(L, Gd, nz) as pl:
        y1 = pl.apply(x1, False)
        y2 = pl.apply(x2, False)
        y3 = pl.apply(x3, True)
        y4 = pl.apply(x1, False)
        for y, x, adj, what in ((y1, x1, False, "x1"), (y2, x2, False, "x2"), (y3, x3, True, "adjoint"),
                                (y4, x1, False, "x1 again")):
            fredholm_check(Gd, x, y, adj, what)
        assert torch.equal(bits(torch.view_as_real(y4) if cx else y4), bits(torch.view_as_real(y1) if cx else y1))


def peer_outputs(nfloat, npeers, y_off):
    """guarded flat float32 buffers for y (at element offset y_off) and npeers peer outputs (16-byte aligned)"""
    return guarded(1, nfloat, nfloat, y_off), [guarded(1, nfloat, nfloat, 4) for _ in range(npeers)]


@pytest.mark.parametrize("cx", [False, True])
def test_fredholm_tc_peer_epilogue(L, cx):
    """the fused all-gather epilogue on one GPU: three local buffers stand in for the peers.  y and every peer hold
    the same bits; a y one float off 8-byte alignment (scalar stores) gives the same bits as the aligned one"""
    rng = np.random.default_rng(600 + 2 * cx)
    nsl, nx, ny, nz = 3, 70, 90, 40
    Gd = to_dev(sign_unit(rng, (nsl, nx, ny), cx), cx)
    with FredholmPlan(L, Gd, nz) as pl:
        for adjoint in (False, True):
            m, K = (ny, nx) if adjoint else (nx, ny)
            xd = to_dev(sign_unit(rng, (nsl, K, nz), cx) * 2.0 ** distinct_pow2(rng, nz)[None, None, :], cx)
            nf = nsl * m * nz * (2 if cx else 1)
            outs = {}
            for y_off in (4, 5):
                (ybuf, yv), peers = peer_outputs(nf, 3, y_off)
                L.check(L.lib.b2_fredholm_apply(pl.h, xd.data_ptr(), yv.data_ptr(),
                                                ptr_array([p.data_ptr() for _, p in peers]), 3, int(adjoint),
                                                L.stream()), "b2_fredholm_apply")
                assert guards_intact(ybuf, yv), f"store outside y, offset {y_off}"
                for i, (pbuf, pv) in enumerate(peers):
                    assert torch.equal(bits(pv), bits(yv)), f"peer {i}, y offset {y_off}"
                    assert guards_intact(pbuf, pv), f"store outside peer {i}, y offset {y_off}"
                outs[y_off] = yv.clone()
            assert torch.equal(bits(outs[4]), bits(outs[5])), f"scalar stores differ, adjoint={adjoint}"
            y = outs[4].view(-1).view(torch.complex64) if cx else outs[4].view(-1)
            fredholm_check(Gd, xd, y.view(nsl, m, nz), adjoint, f"adjoint={adjoint}")


@pytest.mark.parametrize("dt", ["f32", "c64", "f64"])
def test_batched_gemm_allgather_peers(L, dt):
    """SIMT product + fused all-gather on one GPU: y and three local 'peer' buffers are bit-identical to the plain
    batched product, with nothing stored outside them"""
    npdt, code = DT[dt]
    rng = np.random.default_rng(700 + code)
    nsl, nx, ny, nz = 5, 37, 45, 19
    esz = np.dtype(npdt).itemsize // 4
    Gd = dev(rnd(rng, nsl * nx * ny, npdt))
    for adjoint in (0, 1):
        m, K = (ny, nx) if adjoint else (nx, ny)
        xd = dev(rnd(rng, nsl * K * nz, npdt))
        plain = torch.empty(nsl * m * nz, dtype=xd.dtype, device="cuda")
        L.check(L.lib.b2_batched_gemm(L.ctx(), Gd.data_ptr(), xd.data_ptr(), plain.data_ptr(), nsl, nx, ny, nz, adjoint,
                                      code, L.stream()))
        nf = nsl * m * nz * esz
        (ybuf, yv), peers = peer_outputs(nf, 3, 4)
        L.check(L.lib.b2_batched_gemm_allgather(L.ctx(), Gd.data_ptr(), xd.data_ptr(), yv.data_ptr(),
                                                ptr_array([p.data_ptr() for _, p in peers]), 3, nsl, nx, ny, nz,
                                                adjoint, code, L.stream()), "b2_batched_gemm_allgather")
        assert torch.equal(bits(yv.reshape(-1)), bits(plain.view(torch.float32))), f"adjoint={adjoint}"
        assert guards_intact(ybuf, yv)
        for i, (pbuf, pv) in enumerate(peers):
            assert torch.equal(bits(pv), bits(yv)), f"peer {i} adjoint={adjoint}"
            assert guards_intact(pbuf, pv), f"store outside peer {i}"


@pytest.mark.gpu
def test_c_abi_client(tmp_path):
    """plain-C99 program (tests/abi/abi_smoke.c) drives the host-buffer plugin entry point through the C ABI"""
    import subprocess
    from test_host_logic import _build_c_client
    exe = _build_c_client(tmp_path)
    res = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "max |err|" in res.stdout
