"""Return codes of the entry points that choose their kernels by a dtype code.

Every entry point is called through the C ABI with each dtype code from -1 to 7, with an empty and a non-empty size,
and with a null pointer where it checks for one.  The expected code follows the order of the entry point's checks:
a null pointer, a size of zero and a bad dtype each win over the others in the order the header documents, and
that order is what callers see.  Every call that passes its checks launches on valid, zero-filled device memory.
"""
import ctypes as C
from types import SimpleNamespace

import pytest
import torch

OK, DTYPE, ARG, UNSUPPORTED = 0, 2001, 2002, 2005
CUDA_INVALID_CONFIGURATION = 9   # cudaErrorInvalidConfiguration: a launch with a zero grid dimension
CODES = range(-1, 8)
ALL = (0, 1, 2, 3)               # F32, F64, C64, C128
REAL = (0, 1)                    # F32, F64
N = 16                           # elements of a non-empty call


def dt(d, ok=ALL):
    return OK if d in ok else DTYPE


ENTRIES = {}


def entry(f):
    ENTRIES[f.__name__] = f
    return f


@entry
def b2_lincomb(L, p):
    a_re, a_cx, b = L.cpair(2.0), L.cpair(2.0 - 1.0j), L.cpair(0.5)
    for d in CODES:
        for n in (0, N):
            for a, y, conj in ((a_re, p.y, 0), (a_re, None, 0), (a_cx, p.y, 0), (a_re, p.y, 1), (a_cx, None, 1)):
                rc = L.lib.b2_lincomb(p.ctx, p.z, a, p.x, b, y, n, d, conj, p.st)
                yield (d, n, a[1], y is None, conj), rc, dt(d)
        yield (d, "x NULL"), L.lib.b2_lincomb(p.ctx, p.z, a_re, None, b, p.y, N, d, 0, p.st), ARG


@entry
def b2_lincomb_dev(L, p):
    for d in CODES:
        for n in (0, N):
            yield (d, n), L.lib.b2_lincomb_dev(p.ctx, p.z, p.coef, 2.0, p.x, None, 0.0, None, n, d, p.st), dt(d)
            rc = L.lib.b2_lincomb_dev(p.ctx, p.z, p.coef, 2.0, p.x, p.coef, 0.5, p.y, n, d, p.st)
            yield (d, n, "y"), rc, dt(d)
        yield (d, "x NULL"), L.lib.b2_lincomb_dev(p.ctx, p.z, p.coef, 2.0, None, None, 0.0, None, N, d, p.st), ARG


@entry
def b2_mul(L, p):
    for d in CODES:
        for n in (0, N):
            for conj in (0, 1):
                yield (d, n, conj), L.lib.b2_mul(p.ctx, p.z, p.x, p.y, n, d, conj, p.st), OK if n == 0 else dt(d)
        yield (d, "y NULL"), L.lib.b2_mul(p.ctx, p.z, p.x, None, N, d, 0, p.st), ARG


@entry
def b2_fill(L, p):
    v = L.cpair(1.0 + 2.0j)
    for d in CODES:
        for n in (0, N):
            yield (d, n), L.lib.b2_fill(p.ctx, p.z, v, n, d, p.st), OK if n == 0 else dt(d)
        yield (d, "v NULL"), L.lib.b2_fill(p.ctx, p.z, None, N, d, p.st), ARG


@entry
def b2_gemv(L, p):
    for d in CODES:
        for op in (0, 1, 2):
            for m, n in ((0, 0), (4, 0), (0, 4), (4, 4)):
                in_len = n if op == 0 else m      # an empty contraction clears y before the dtype is looked at
                want = OK if (m == 0 and n == 0) or in_len == 0 else dt(d)
                yield (d, op, m, n), L.lib.b2_gemv(p.ctx, p.x, 4, m, n, p.y, p.z, op, d, d, p.st), want
            yield (d, op, "A NULL"), L.lib.b2_gemv(p.ctx, None, 4, 4, 4, p.y, p.z, op, d, d, p.st), ARG
        # bf16 A takes float32 x and y only; any other pair of codes must be equal
        yield (4, d), L.lib.b2_gemv(p.ctx, p.x, 8, 4, 8, p.y, p.z, 0, 4, d, p.st), OK if d == 0 else DTYPE
        if d in ALL:
            yield (d, d ^ 1), L.lib.b2_gemv(p.ctx, p.x, 4, 4, 4, p.y, p.z, 0, d, d ^ 1, p.st), DTYPE


@entry
def b2_gemm(L, p):
    for d in CODES:
        for op in (0, 1, 2):
            for m, n, k in ((0, 4, 4), (4, 0, 4), (4, 4, 0), (4, 4, 4)):
                for acc in (0, 1):
                    rc = L.lib.b2_gemm(p.ctx, p.x, 4, p.y, 4, p.z, 4, m, n, k, op, acc, d, p.st)
                    yield (d, op, m, n, k, acc), rc, dt(d)
        yield (d, "A NULL"), L.lib.b2_gemm(p.ctx, None, 4, p.y, 4, p.z, 4, 4, 4, 4, 0, 0, d, p.st), ARG
        yield (d, "A NULL, m 0"), L.lib.b2_gemm(p.ctx, None, 4, p.y, 4, p.z, 4, 0, 4, 4, 0, 0, d, p.st), dt(d)
        yield (d, "C NULL"), L.lib.b2_gemm(p.ctx, p.x, 4, p.y, 4, None, 4, 4, 4, 0, 0, 0, d, p.st), ARG


@entry
def b2_batched_gemm(L, p):
    for d in CODES:
        for nsl in (0, 2):
            for adj in (0, 1):
                for nx, ny, nz in ((4, 4, 4), (0, 4, 4), (4, 0, 4), (4, 4, 0)):
                    rc = L.lib.b2_batched_gemm(p.ctx, p.x, p.y, p.z, nsl, nx, ny, nz, adj, d, p.st)
                    yield (d, nsl, adj, nx, ny, nz), rc, OK if nsl == 0 else dt(d)
            yield (d, nsl, "G NULL"), L.lib.b2_batched_gemm(p.ctx, None, p.y, p.z, nsl, 4, 4, 4, 0, d, p.st), \
                OK if nsl == 0 else ARG


@entry
def b2_batched_gemm_allgather(L, p):
    for d in CODES:
        for nsl in (0, 2):
            for adj in (0, 1):
                for nx, ny, nz in ((4, 4, 4), (0, 4, 4), (4, 0, 4), (4, 4, 0)):
                    m = ny if adj else nx
                    rc = L.lib.b2_batched_gemm_allgather(p.ctx, p.x, p.y, p.z, None, 0, nsl, nx, ny, nz, adj, d, p.st)
                    # the fused product leaves an empty output grid to the launch, which reports it
                    want = OK if nsl == 0 else dt(d) if d not in ALL or (m and nz) else CUDA_INVALID_CONFIGURATION
                    yield (d, nsl, adj, nx, ny, nz), rc, want
            rc = L.lib.b2_batched_gemm_allgather(p.ctx, p.x, None, p.z, None, 0, nsl, 4, 4, 4, 0, d, p.st)
            yield (d, nsl, "x NULL"), rc, OK if nsl == 0 else ARG


@entry
def b2_dot(L, p):
    for d in CODES:
        for n in (0, N):
            for conj in (0, 1):
                p.res.fill_(7.0)
                yield (d, n, conj), L.lib.b2_dot(p.ctx, p.x, p.y, n, d, conj, p.out, p.st), dt(d)
                # the imaginary slot is cleared for every code but C64 / C128, before the code is rejected
                yield (d, n, conj, "imag"), float(p.res[1]), 0.0
        yield (d, "x NULL"), L.lib.b2_dot(p.ctx, None, p.y, N, d, 0, p.out, p.st), ARG
        yield (d, "x NULL, n 0"), L.lib.b2_dot(p.ctx, None, None, 0, d, 0, p.out, p.st), dt(d)


@entry
def b2_norm_partial(L, p):
    for d in CODES:
        for n in (0, N):
            for kind, pw in ((2, 2.0), (3, 0.0), (5, 1.5), (99, 0.0)):
                rc = L.lib.b2_norm_partial(p.ctx, p.x, n, d, kind, pw, p.out, p.st)
                yield (d, n, kind), rc, ARG if kind == 99 else dt(d)
        yield (d, "x NULL"), L.lib.b2_norm_partial(p.ctx, None, N, d, 2, 2.0, p.out, p.st), ARG


@entry
def b2_dot_multi(L, p):
    xs, ys = (C.c_void_p * 2)(p.x, p.y), (C.c_void_p * 2)(p.y, p.x)
    for d in CODES:
        for n in (0, N):
            for conj in (0, 1):
                yield (d, n, conj), L.lib.b2_dot_multi(p.ctx, 2, xs, ys, n, d, conj, p.out, p.st), dt(d)
            yield (d, n, "k 5"), L.lib.b2_dot_multi(p.ctx, 5, xs, ys, n, d, 0, p.out, p.st), ARG
        yield (d, "xs NULL"), L.lib.b2_dot_multi(p.ctx, 2, None, ys, N, d, 0, p.out, p.st), ARG


@entry
def b2_sparse_update(L, p):
    for d in CODES:
        for n in (0, N):
            for kind in (0, 1, 2, 3):
                for base in (p.x, None):
                    rc = L.lib.b2_sparse_update(p.ctx, base, p.y, 0.5, None, 0.1, kind, p.z, None, 0.0, p.out, n, d,
                                                p.st)
                    want = (UNSUPPORTED if kind == 3 and d in (2, 3) else DTYPE if d not in ALL
                            else ARG if base is None and n else OK)
                    yield (d, n, kind, base is None), rc, want


@entry
def b2_lsqr_update(L, p):
    for d in CODES:
        for n in (0, N):
            for var in (None, p.w):
                for x in (p.x, None):
                    rc = L.lib.b2_lsqr_update(p.ctx, x, p.y, p.z, var, n, d, p.coef, None, p.out, p.st)
                    yield (d, n, var is None, x is None), rc, DTYPE if d not in ALL else ARG if x is None and n else OK


@entry
def b2_derivative_axis(L, p):
    for d in CODES:
        for n_axis in (0, 8):
            for deriv in (1, 2):
                rc = L.lib.b2_derivative_axis(p.ctx, p.x, p.z, 2, n_axis, 32, deriv, 2, 3, 0, 1.0, 0, d, p.st)
                yield (d, n_axis, deriv), rc, OK if n_axis == 0 else dt(d, REAL)
        yield (d, "x NULL"), L.lib.b2_derivative_axis(p.ctx, None, p.z, 2, 8, 32, 1, 2, 3, 0, 1.0, 0, d, p.st), ARG


@entry
def b2_first_derivative(L, p):
    for d in CODES:
        for nloc in (0, 8):
            for ncols in (32, 3):
                rc = L.lib.b2_first_derivative(p.ctx, p.x, p.z, None, 0, None, 0, nloc, ncols, 0, nloc, 2, 3, 0, 1.0,
                                               0, d, p.st)
                yield (d, nloc, ncols), rc, OK if nloc == 0 else dt(d, REAL)
            rc = L.lib.b2_second_derivative(p.ctx, p.x, p.z, None, 0, None, 0, nloc, 32, 0, nloc, 2, 0, 1.0, 0, d,
                                            p.st)
            yield (d, nloc, "second"), rc, OK if nloc == 0 else dt(d, REAL)
        rc = L.lib.b2_first_derivative(p.ctx, None, p.z, None, 0, None, 0, 8, 32, 0, 8, 2, 3, 0, 1.0, 0, d, p.st)
        yield (d, "x NULL"), rc, ARG


@entry
def b2_kirchhoff(L, p):
    for d in CODES:
        for ni in (0, 64):
            for adj in (0, 1):
                rc = L.lib.b2_kirchhoff(p.ctx, p.x, p.z, p.coef, p.coef, ni, 1, 1, 8, 1.0, adj, d, p.st)
                yield (d, ni, adj), rc, ARG if ni == 0 else dt(d, REAL)
            for nc in (0, 32):
                rc = L.lib.b2_kirchhoff_chunk(p.ctx, p.x, p.z, p.coef, p.coef, 64, 32, nc, 1, 1, 8, 1.0, 0, 0, d, p.st)
                yield (d, "chunk", nc), rc, ARG if nc == 0 else dt(d, REAL)
        yield (d, "x NULL"), L.lib.b2_kirchhoff(p.ctx, None, p.z, p.coef, p.coef, 64, 1, 1, 8, 1.0, 0, d, p.st), ARG


@entry
def b2_convolve_axis(L, p):
    for d in CODES:
        for n_axis in (0, 8):
            for n_inner in (1, 4):
                for adj in (0, 1):
                    rc = L.lib.b2_convolve_axis(p.ctx, p.x, p.z, 2, n_axis, n_inner, p.coef, 3, 1, adj, d, p.st)
                    yield (d, n_axis, n_inner, adj), rc, dt(d, REAL)
                    for kind in (0, 1, 2):
                        rc = L.lib.b2_poststack_axis(p.ctx, p.x, p.z, 2, n_axis, n_inner, p.coef, 3, 1, kind, adj, d,
                                                     p.st)
                        yield (d, n_axis, n_inner, adj, kind), rc, ARG if kind == 1 else dt(d, REAL)
            # the dtype is checked before the block is found empty, and both before x
            rc = L.lib.b2_convolve_axis(p.ctx, None, p.z, 2, n_axis, 4, p.coef, 3, 1, 0, d, p.st)
            yield (d, n_axis, "x NULL"), rc, DTYPE if d not in REAL else OK if n_axis == 0 else ARG


@entry
def b2_nsconvolve_axis(L, p):
    for d in CODES:
        for n_axis in (0, 8):
            for n_inner in (1, 4):
                for adj in (0, 1):
                    rc = L.lib.b2_nsconvolve_axis(p.ctx, p.x, p.z, 2, n_axis, n_inner, p.coef, 2, 3, 1, 0, 4, adj, d,
                                                  p.st)
                    yield (d, n_axis, n_inner, adj), rc, ARG if n_axis == 0 else dt(d, REAL)
                    for kind in (0, 1, 2):
                        rc = L.lib.b2_nspoststack_axis(p.ctx, p.x, p.z, 2, n_axis, n_inner, p.coef, 2, 3, 1, 0, 4,
                                                       kind, adj, d, p.st)
                        yield (d, n_axis, n_inner, adj, kind), rc, ARG if n_axis == 0 or kind == 1 else dt(d, REAL)
        rc = L.lib.b2_nsconvolve_axis(p.ctx, None, p.z, 2, 8, 4, p.coef, 2, 3, 1, 0, 4, 0, d, p.st)
        yield (d, "x NULL"), rc, ARG


@pytest.fixture(scope="module")
def L():
    import pylops_mpi_b200._lib as L
    return L


@pytest.fixture(scope="module")
def p(L):
    # 64 KB of zeros per array: more than any call below reads or writes, in any dtype
    buf = [torch.zeros(8192, dtype=torch.float64, device="cuda") for _ in range(6)]
    x, y, z, w, coef, res = buf
    return SimpleNamespace(ctx=L.ctx(), st=L.stream(), x=x.data_ptr(), y=y.data_ptr(), z=z.data_ptr(),
                           w=w.data_ptr(), coef=coef.data_ptr(), out=res.data_ptr(), res=res)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ENTRIES))
def test_return_codes(L, p, name):
    bad = [(case, rc, want) for case, rc, want in ENTRIES[name](L, p) if rc != want]
    torch.cuda.synchronize()
    assert not bad, f"{name}: (case, got, want) {bad}"
