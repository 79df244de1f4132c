"""Dense SIMT products past their launch limits: the transposed gemv past the ticket budget of its column tiles
(4032 tiles) and past 65535 row chunks of 128 rows, the SIMT product past 65535 row tiles of 64 rows, the batched
product past 65535 slices, pitched operands, and the transposed gemv's chunk-partial scratch under CUDA graphs.

At every shape at or past a limit the data are small integers ({-1, 0, 1} in A, small integers in x, in the real and
imaginary parts alike), so that every partial sum stays below 2^24: the float32 and float64 kernels must then EQUAL
the float64 reference bit for bit, in any summation order, and a dropped, doubled or misplaced row, chunk or column
tile fails loudly.  Where rounding matters, the tolerance is derived from the longest serial accumulation chain of
the kernel at that shape (stated at each use)."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

B2_ERR_WORKSPACE = 2004
TICKET_TILES = 4096 - 64          # column tiles one multi-chunk transposed gemv launch can hold
GT_ROWS = 128                     # rows of a transposed-gemv chunk while m <= 65535 * 128
GRID_Y = 65535
GEMM_ROWS = GRID_Y * 64           # output rows of one SIMT product launch
A_BYTES_MAX = 320 * 2 ** 20       # largest A a case allocates

# name -> (torch dtype of A, torch dtype of x / y, code of A, code of x / y, elements of A per 16 bytes)
DT = {"f32": (torch.float32, torch.float32, 0, 0, 4), "f64": (torch.float64, torch.float64, 1, 1, 2),
      "c64": (torch.complex64, torch.complex64, 2, 2, 2), "c128": (torch.complex128, torch.complex128, 3, 3, 1),
      "bf16": (torch.bfloat16, torch.float32, 4, 0, 8)}
U = {torch.float32: 2.0 ** -24, torch.complex64: 2.0 ** -24, torch.float64: 2.0 ** -53, torch.complex128: 2.0 ** -53}


@pytest.fixture(scope="module")
def L():
    import pylops_mpi_b200._lib as L
    yield L
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


def ints(shape, dtype, lo, hi, gen):
    """integers in [lo, hi] of ``dtype`` on the device (complex: in the real and the imaginary part)"""
    def part():
        return torch.randint(lo, hi + 1, shape, generator=gen, device="cuda", dtype=torch.int8)
    if dtype.is_complex:
        return torch.complex(part().to(torch.float64), part().to(torch.float64)).to(dtype)
    return part().to(dtype)


def wide(t):
    """float64 / complex128 copy (exact for every dtype here)"""
    return t.to(torch.complex128 if t.dtype.is_complex else torch.float64)


def bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(torch.view_as_real(a).view(torch.uint8)
                                                                     if a.is_complex() else a.view(torch.uint8),
                                                                     torch.view_as_real(b).view(torch.uint8)
                                                                     if b.is_complex() else b.view(torch.uint8))


def gamma(n, u):
    """Higham's gamma_n = n u / (1 - n u): the relative error bound of n chained roundings"""
    return n * u / (1 - n * u)


def chunk_rows(m):
    """rows per chunk of the transposed gemv: 128, or the multiple of 128 that keeps the chunks within 65535"""
    return GT_ROWS * (-(-m // (GT_ROWS * GRID_Y)))


def padded(m, n, lda, dtype, gen, lo=-1, hi=1):
    """(m x lda buffer, its m x n view): integer entries, NaN in the pitch padding (a read of it poisons y)"""
    buf = torch.empty((m, lda), dtype=dtype, device="cuda")
    buf[:, :n] = ints((m, n), dtype, lo, hi, gen)
    if lda > n:
        buf[:, n:] = float("nan")
    return buf, buf[:, :n]


def gemv(L, A, lda, m, n, x, y, op, dt, ctx=None, stream=None):
    _, _, ca, cx, _ = DT[dt]
    return L.lib.b2_gemv(ctx or L.ctx(), A.data_ptr(), lda, m, n, x.data_ptr(), y.data_ptr(), op, ca, cx,
                         stream if stream is not None else L.stream())


def run_gemv_t(L, A, lda, m, n, x, op, dt):
    """y = op(A) x for op T / H, y written into a buffer with a sentinel tail that must stay untouched"""
    xdt = DT[dt][1]
    ybuf = torch.full((n + 67,), 12345.0, dtype=xdt, device="cuda")
    L.check(gemv(L, A, lda, m, n, x, ybuf, op, dt), "b2_gemv")
    assert torch.all(ybuf[n:] == 12345.0), "transposed gemv wrote past y"
    return ybuf[:n]


def op_t(A64, op):
    return A64.conj().T if op == 2 else A64.T


def probes(m, extra=()):
    rows = chunk_rows(m)
    last = (m - 1) // rows * rows                     # first row of the last chunk
    cand = {0, m - 1, 127, 128, 129, last, last - 1, last + 1, m - GT_ROWS, m - GT_ROWS - 1, *extra}
    return sorted(i for i in cand if 0 <= i < m)


def check_one_hot(L, A, lda, m, n, op, dt, rows):
    """x = e_i: the result must be exactly row i of A (conjugated for op H)"""
    xdt = DT[dt][1]
    x = torch.zeros(m, dtype=xdt, device="cuda")
    for i in rows:
        x.zero_()
        x[i] = 1
        y = run_gemv_t(L, A, lda, m, n, x, op, dt)
        row = A[i, :n].to(xdt)
        want = row.conj().resolve_conj() if op == 2 else row
        assert torch.equal(y, want), f"one-hot probe row {i} of {m}"


# ------------------------------------------------------------------------------------------------------------------
# a. transposed gemv past the ticket budget of its column tiles
# ------------------------------------------------------------------------------------------------------------------
def _ticket_cases():
    cases = []
    for dt, (adt, _, _, _, V) in DT.items():
        esz = torch.empty((), dtype=adt).element_size()
        for layout in ("vec", "scalar"):
            if layout == "scalar" and esz == 16:
                continue                      # a complex128 row pitch is always a multiple of 16 bytes
            tile = 32 * (V if layout == "vec" else 1)
            lim = TICKET_TILES * tile
            for n in (lim, lim + 1, lim + 3 * tile + 5):
                if layout == "vec":
                    lda = -(-n // V) * V      # multiple of 16 bytes; > n when n is ragged
                else:
                    lda = n + 1 if ((n + 1) * esz) % 16 else n + 2
                for m in (1, 128, 129, 1000):
                    if m * lda * esz <= A_BYTES_MAX:
                        cases.append(pytest.param(dt, layout, m, n, lda, id=f"{dt}-{layout}-m{m}-n{n}"))
    return cases


@pytest.mark.parametrize("dt,layout,m,n,lda", _ticket_cases())
def test_gemv_t_past_ticket_budget_exact(L, dt, layout, m, n, lda):
    adt, xdt = DT[dt][0], DT[dt][1]
    gen = torch.Generator(device="cuda").manual_seed(m * 7 + n)
    buf, A = padded(m, n, lda, adt, gen)
    A64 = wide(A)
    for op in (1, 2):
        x = ints((m,), xdt, -3, 3, gen)
        y = run_gemv_t(L, buf, lda, m, n, x, op, dt)
        ref = op_t(A64, op) @ wide(x)
        assert torch.equal(wide(y), ref)
        if m > 1:
            check_one_hot(L, buf, lda, m, n, op, dt, probes(m))


# ------------------------------------------------------------------------------------------------------------------
# b. transposed gemv past 65535 row chunks
# ------------------------------------------------------------------------------------------------------------------
TALL_M = (GRID_Y * GT_ROWS, GRID_Y * GT_ROWS + 1, 9_000_001)


@pytest.mark.parametrize("m", TALL_M)
@pytest.mark.parametrize("dt,n", [("f32", 1), ("f32", 5), ("f64", 2), ("c128", 1)])
def test_gemv_t_past_chunk_limit_exact(L, m, dt, n):
    adt, xdt = DT[dt][0], DT[dt][1]
    gen = torch.Generator(device="cuda").manual_seed(m + n)
    A = ints((m, n), adt, -1, 1, gen)
    A64 = wide(A)
    for op in (1, 2):
        x = ints((m,), xdt, -1, 1, gen)              # |partial sums| <= m < 2^24
        y = run_gemv_t(L, A, n, m, n, x, op, dt)
        assert torch.equal(wide(y), op_t(A64, op) @ wide(x))
        rows = chunk_rows(m)
        nch = -(-m // rows)
        check_one_hot(L, A, n, m, n, op, dt, probes(m, ((nch - 2) * rows, (nch - 1) * rows - 1,
                                                        (GRID_Y - 1) * GT_ROWS, (GRID_Y - 1) * GT_ROWS - 1)))


# ------------------------------------------------------------------------------------------------------------------
# c. a transposed gemv called twice gives the same bits (the last CTA of each tile resets its ticket)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt,m,n,lda", [
    ("f32", 129, 2 * 129_024 + 7, 2 * 129_024 + 9),      # scalar layout, 3 launches of column tiles
    ("c64", 129, 2 * 129_024 + 3, 2 * 129_024 + 3),      # row pitch 8 * odd bytes: scalar layout, 3 launches
    ("bf16", 300, 2 * 129_024 + 40, 2 * 129_024 + 41),   # scalar layout, 3 launches, 3 chunks
    ("f64", 257, 258_048 + 2, 258_048 + 2),              # vector layout, 2 launches
    ("f32", GRID_Y * GT_ROWS + 1, 1, 1),                 # 256-row chunks
])
def test_gemv_t_repeat_is_bit_identical(L, dt, m, n, lda):
    adt, xdt = DT[dt][0], DT[dt][1]
    torch.manual_seed(m + n)
    buf = torch.randn((m, lda), device="cuda", dtype=torch.complex128 if adt.is_complex else torch.float64).to(adt)
    x = torch.randn(m, device="cuda", dtype=torch.complex128 if xdt.is_complex else torch.float64).to(xdt)
    for op in (1, 2):
        y1 = run_gemv_t(L, buf, lda, m, n, x, op, dt).clone()
        y2 = run_gemv_t(L, buf, lda, m, n, x, op, dt)
        assert bits_equal(y1, y2)
        check_rounded_gemv_t(buf[:, :n], x, y1, op, xdt)


def check_rounded_gemv_t(A, x, y, op, xdt):
    """|y - op(A) x| <= (gamma_h(u) + gamma_m(2^-53)) * c * (|A|^T |x|), h the longest serial chain of the kernel:
    ceil(rows / 8) fma per lane and chunk (2 per row for complex), 7 adds folding the 8 warps, nchunks - 1 adds
    folding the chunks in order, 1 to spare; gamma_m for the float64 reference; c = 2 for complex (re and im parts
    each bounded by sum |a| |x|)"""
    m = A.shape[0]
    rows = chunk_rows(m)
    nch = -(-m // rows)
    cx = xdt.is_complex
    h = (2 if cx else 1) * (-(-rows // 8)) + 7 + (nch - 1) + 1
    A64, x64 = wide(A), wide(x)
    ref = op_t(A64, op) @ x64
    mag = A64.abs().T @ x64.abs()
    tol = (gamma(h, U[xdt]) + gamma(m, 2.0 ** -53)) * (2 if cx else 1) * mag
    err = (wide(y) - ref).abs()
    assert torch.all(err <= tol), float((err / tol.clamp_min(1e-300)).max())


# ------------------------------------------------------------------------------------------------------------------
# d. SIMT product past 65535 row tiles
# ------------------------------------------------------------------------------------------------------------------
def gemm(L, A, lda, B, ldb, Cm, ldc, m, n, k, op, acc, code):
    return L.lib.b2_gemm(L.ctx(), A.data_ptr(), lda, B.data_ptr(), ldb, Cm.data_ptr(), ldc, m, n, k, op, acc, code,
                         L.stream())


def check_gemm_exact(L, m, n, k, dt, gen, ops=(0, 1, 2)):
    adt = DT[dt][0]
    code = DT[dt][2]
    B = ints((k, n), adt, -3, 3, gen)
    C0 = ints((m, n), adt, -3, 3, gen)
    for op in ops:
        A = ints((m, k) if op == 0 else (k, m), adt, -1, 1, gen)
        opA = wide(A) if op == 0 else op_t(wide(A), op)
        prod = opA @ wide(B)
        del opA
        for acc in (0, 1):
            Cm = C0.clone()
            L.check(gemm(L, A, A.shape[1], B, n, Cm, n, m, n, k, op, acc, code), "b2_gemm")
            want = prod + wide(C0) if acc else prod
            assert torch.equal(wide(Cm), want), (op, acc)
        del A, prod


@pytest.mark.parametrize("m", [GEMM_ROWS, GEMM_ROWS + 1, 4_300_001])
@pytest.mark.parametrize("k", [1, 17])
def test_gemm_simt_past_grid_rows_exact_f32(L, m, k):
    gen = torch.Generator(device="cuda").manual_seed(m + k)
    for n in (1, 3):
        check_gemm_exact(L, m, n, k, "f32", gen)


@pytest.mark.parametrize("dt", ["f64", "c128"])
def test_gemm_simt_past_grid_rows_exact_wide_types(L, dt):
    check_gemm_exact(L, GEMM_ROWS + 1, 2, 3, dt, torch.Generator(device="cuda").manual_seed(3))


# ------------------------------------------------------------------------------------------------------------------
# e. SIMT product with pitched operands
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt,m,n,k", [(dt, m, n, k) for dt in ("f32", "f64", "c64", "c128")
                                        for m, n, k in ((130, 70, 33), (1, 1, 2), (65, 129, 17))]
                         + [("f32", GEMM_ROWS + 70, 3, 2)])
def test_gemm_simt_pitched_operands(L, dt, m, n, k):
    """lda, ldb, ldc past the row lengths: NaN in A's and B's padding (read, it would poison C), a sentinel in C's
    padding columns that must survive; the tall case has several launches of row groups"""
    adt, code = DT[dt][0], DT[dt][2]
    gen = torch.Generator(device="cuda").manual_seed(m * 3 + n)
    ldb, ldc = n + 3, n + 5
    Bbuf, B = padded(k, n, ldb, adt, gen, -3, 3)
    for op in (0, 1, 2):
        ar, ac = (m, k) if op == 0 else (k, m)
        Abuf, A = padded(ar, ac, ac + 7, adt, gen)
        opA = wide(A) if op == 0 else op_t(wide(A), op)
        prod = opA @ wide(B)
        del opA
        for acc in (0, 1):
            Cbuf = torch.full((m, ldc), 777.0, dtype=adt, device="cuda")
            C0 = ints((m, n), adt, -3, 3, gen)
            Cbuf[:, :n] = C0
            L.check(gemm(L, Abuf, ac + 7, Bbuf, ldb, Cbuf, ldc, m, n, k, op, acc, code), "b2_gemm")
            want = prod + wide(C0) if acc else prod
            assert torch.equal(wide(Cbuf[:, :n]), want), (op, acc)
            assert torch.all(Cbuf[:, n:] == 777.0), "padding columns of C were written"
        del Abuf, A, prod


# ------------------------------------------------------------------------------------------------------------------
# f. batched product across its 65535-slice launches
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nsl", [GRID_Y, GRID_Y + 1, GRID_Y + 3])
@pytest.mark.parametrize("dt", ["f32", "f64", "c64", "c128"])
@pytest.mark.parametrize("adjoint", [0, 1])
def test_batched_gemm_past_slice_limit_exact(L, nsl, dt, adjoint):
    adt, code = DT[dt][0], DT[dt][2]
    nx, ny, nz = 3, 2, 2
    gen = torch.Generator(device="cuda").manual_seed(nsl + adjoint)
    G = ints((nsl, nx, ny), adt, -3, 3, gen)
    x = ints((nsl, nx if adjoint else ny, nz), adt, -3, 3, gen)
    rows = ny if adjoint else nx
    ybuf = torch.full((nsl * rows * nz + 16,), 777.0, dtype=adt, device="cuda")
    L.check(L.lib.b2_batched_gemm(L.ctx(), G.data_ptr(), x.data_ptr(), ybuf.data_ptr(), nsl, nx, ny, nz, adjoint,
                                  code, L.stream()), "b2_batched_gemm")
    G64 = wide(G)
    ref = (G64.conj().transpose(1, 2) if adjoint else G64) @ wide(x)
    assert torch.equal(wide(ybuf[:nsl * rows * nz].view(nsl, rows, nz)), ref)
    assert torch.all(ybuf[nsl * rows * nz:] == 777.0)


# ------------------------------------------------------------------------------------------------------------------
# g. rounding-realistic data: random normal, tolerance from the longest serial accumulation chain
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", ["f32", "f64", "c64", "c128"])
def test_gemm_simt_deep_k_rounding(L, dt):
    """m, n ragged across the 64-tiles, k = 4099 = 256 K-slices of 16 plus a ragged one.  Each output element is
    ONE thread's serial fma chain over k (2 k for complex: re and im take two fma each per term), so
    |C - op(A) B| <= (gamma_{c k}(u) + gamma_k(2^-53)) * c * (|op(A)| |B|), the second term for the float64
    reference, c = 2 for complex"""
    adt, code = DT[dt][0], DT[dt][2]
    m, n, k = 193, 131, 4099
    cx = adt.is_complex
    w = torch.complex128 if cx else torch.float64
    torch.manual_seed(7)
    B = torch.randn((k, n), dtype=w, device="cuda").to(adt)
    for op in (0, 1, 2):
        A = torch.randn((m, k) if op == 0 else (k, m), dtype=w, device="cuda").to(adt)
        Cm = torch.empty((m, n), dtype=adt, device="cuda")
        L.check(gemm(L, A, A.shape[1], B, n, Cm, n, m, n, k, op, 0, code), "b2_gemm")
        opA = wide(A) if op == 0 else op_t(wide(A), op)
        ref = opA @ wide(B)
        mag = opA.abs() @ wide(B).abs()
        c = 2 if cx else 1
        tol = (gamma(c * k, U[adt]) + gamma(k, 2.0 ** -53)) * c * mag
        err = (wide(Cm) - ref).abs()
        assert torch.all(err <= tol), (op, float((err / tol).max()))


@pytest.mark.parametrize("dt,m,n", [
    ("f32", 130, 520_001), ("f64", 130, 260_001), ("c64", 130, 260_001), ("c128", 130, 130_001),
    ("bf16", 130, 1_040_001),
    ("f32", 8_400_001, 3), ("f64", 8_400_001, 3), ("c64", 8_400_001, 3), ("c128", 8_400_001, 1),
    ("bf16", 8_400_001, 3)])
def test_gemv_t_rounding_wide_and_tall(L, dt, m, n):
    """one shape past the ticket budget and one past the chunk limit per precision; bound: check_rounded_gemv_t"""
    adt, xdt = DT[dt][0], DT[dt][1]
    torch.manual_seed(m + n)
    w = torch.complex128 if adt.is_complex else torch.float64
    A = torch.randn((m, n), dtype=w, device="cuda").to(adt)
    x = torch.randn(m, dtype=w, device="cuda").to(xdt)
    for op in (1, 2):
        y = run_gemv_t(L, A, n, m, n, x, op, dt)
        check_rounded_gemv_t(A, x, y, op, xdt)


# ------------------------------------------------------------------------------------------------------------------
# h. the chunk-partial scratch under CUDA graphs (kernel level, a context of its own)
# ------------------------------------------------------------------------------------------------------------------
def fresh_ctx(L):
    h = C.c_void_p()
    L.check(L.lib.b2_ctx_create(torch.cuda.current_device(), C.byref(h)), "b2_ctx_create")
    return h


def test_gemv_t_graph_survives_scratch_growth(L):
    """a graph captures a 2-chunk transposed gemv; an eager one then needs 32x the chunk-partial bytes; the replay
    (new x) must still be exact: the scratch address the graph holds stays valid.  This pins the contract of the
    grown scratch; it need not fail on a library that frees the old buffer, since the allocator may return the freed
    block inside the new one and the replay then still computes the right y"""
    ctx = fresh_ctx(L)
    g = None
    try:
        gen = torch.Generator(device="cuda").manual_seed(11)
        m, n = 256, 1024                                   # 2 chunks: 8 KB of partials
        A = ints((m, n), torch.float32, -1, 1, gen)
        x = ints((m,), torch.float32, -3, 3, gen)
        y = torch.empty(n, device="cuda")
        L.check(gemv(L, A, n, m, n, x, y, 1, "f32", ctx=ctx), "b2_gemv")      # sizes the scratch
        assert torch.equal(wide(y), wide(A).T @ wide(x))
        g = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            g.capture_begin(capture_error_mode="thread_local")
            try:
                rc = gemv(L, A, n, m, n, x, y, 1, "f32", ctx=ctx, stream=side.cuda_stream)
            finally:
                g.capture_end()
        torch.cuda.current_stream().wait_stream(side)
        L.check(rc, "b2_gemv (captured)")
        mb = 64 * GT_ROWS                                  # 64 chunks: 256 KB of partials, 32x
        Ab = ints((mb, n), torch.float32, -1, 1, gen)
        xb = ints((mb,), torch.float32, -3, 3, gen)
        yb = torch.empty(n, device="cuda")
        L.check(gemv(L, Ab, n, mb, n, xb, yb, 1, "f32", ctx=ctx), "b2_gemv")
        assert torch.equal(wide(yb), wide(Ab).T @ wide(xb))
        x.copy_(ints((m,), torch.float32, -3, 3, gen))
        y.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(wide(y), wide(A).T @ wide(x))
    finally:
        del g
        torch.cuda.synchronize()
        L.check(L.lib.b2_ctx_destroy(ctx), "b2_ctx_destroy")


def test_gemv_t_scratch_growth_during_capture_is_refused(L):
    """growth while the stream captures: B2_ERR_WORKSPACE, nothing enqueued, the capture still ends cleanly"""
    ctx = fresh_ctx(L)
    g = None
    try:
        gen = torch.Generator(device="cuda").manual_seed(12)
        m, n = 256, 100
        A = ints((m, n), torch.float32, -1, 1, gen)
        x = ints((m,), torch.float32, -3, 3, gen)
        y = torch.empty(n, device="cuda")
        g = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            g.capture_begin(capture_error_mode="thread_local")
            try:
                y.fill_(5.0)
                rc = gemv(L, A, n, m, n, x, y, 1, "f32", ctx=ctx, stream=side.cuda_stream)
            finally:
                g.capture_end()
        torch.cuda.current_stream().wait_stream(side)
        assert rc == B2_ERR_WORKSPACE
        y.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.all(y == 5.0), "the refused gemv left a node in the graph"
        # outside the capture the same call grows the scratch and runs
        L.check(gemv(L, A, n, m, n, x, y, 1, "f32", ctx=ctx), "b2_gemv")
        assert torch.equal(wide(y), wide(A).T @ wide(x))
    finally:
        del g
        torch.cuda.synchronize()
        L.check(L.lib.b2_ctx_destroy(ctx), "b2_ctx_destroy")


# ------------------------------------------------------------------------------------------------------------------
# i. the scratch under graphs of operator applies (the package's context, swapped for a fresh one)
# ------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def fresh_package_ctx(L):
    """the package's context of this device replaced by a fresh one for the duration: its chunk-partial scratch
    starts empty, so the sizes below decide when it grows, whatever ran before in the process"""
    dev = torch.cuda.current_device()
    saved = L.ctx(dev)
    h = fresh_ctx(L)
    L._CTX[dev] = h
    try:
        yield h
    finally:
        torch.cuda.synchronize()
        L._CTX[dev] = saved
        L.check(L.lib.b2_ctx_destroy(h), "b2_ctx_destroy")


def test_blockdiag_adjoint_graph_survives_scratch_growth(L, pm):
    """a CUDA graph captures the adjoint of MPIBlockDiag([MatrixMult(A)]) (a 2-chunk transposed gemv, 4 KB of
    partials); the adjoint of a larger MatrixMult then needs 32x those bytes and grows the scratch; replays with new
    data must still be exact.  This pins the scratch contract (a grown scratch keeps the buffer the graph holds).  It
    need not fail on a library that frees the old buffer: the allocator may hand the freed block back inside the new
    one, and the replay then still computes the right y"""
    rng = np.random.default_rng(14)
    nb = 256
    A = np_ints(rng, (nb, nb), np.float64)
    with fresh_package_ctx(L):
        g = None
        try:
            Op = pm.MPIBlockDiag([pm.MatrixMult(A)])
            xd = pm.DistributedArray.to_dist(np_ints(rng, nb, np.float64, -3, 3))
            Op.rmatvec(xd)                                  # eager: loads the kernels, sizes the scratch (4 KB)
            g = torch.cuda.CUDAGraph()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                g.capture_begin(capture_error_mode="thread_local")
                try:
                    yd = Op.rmatvec(xd)
                finally:
                    g.capture_end()
            torch.cuda.current_stream().wait_stream(side)
            big = pm.MatrixMult(torch.ones((16 * GT_ROWS, 1024), dtype=torch.float64, device="cuda"))
            assert torch.all(big.rmatvec(torch.ones(16 * GT_ROWS, dtype=torch.float64, device="cuda")) == 16 * GT_ROWS)
            for _ in range(2):                              # 16 chunks x 1024 columns: 128 KB of partials, 32x
                v = np_ints(rng, nb, np.float64, -3, 3)
                xd.local_array.copy_(torch.as_tensor(v))
                yd.local_array.fill_(float("nan"))
                g.replay()
                torch.cuda.synchronize()
                assert np.array_equal(yd.asarray().cpu().numpy(), A.T @ v)
        finally:
            del g
            torch.cuda.synchronize()


def test_cgls_runs_split_by_larger_adjoint(L, pm):
    """CGLS captures its iteration at the start of each run() and drops the graph at its end, so no solver graph
    outlives a run: a scratch growth between two runs (here certain, the context starts empty) meets no live solver
    graph.  A solve split in two runs with a much larger adjoint between them must equal the float64 oracle run for
    the same total iterations, each run replaying its own graph (graph_replays counts per run)"""
    import pylops_mpi_oracle as o
    rng = np.random.default_rng(13)
    nb = 256
    A = rng.standard_normal((nb, nb)) / 64 + 2 * np.eye(nb)          # singular values in about [1.5, 2.5]
    xt = rng.standard_normal(nb)
    with fresh_package_ctx(L):
        Op = pm.MPIBlockDiag([pm.MatrixMult(A)])
        y = Op @ pm.DistributedArray.to_dist(xt)
        solver = pm.CGLS(Op)
        x = solver.setup(y=y, x0=pm.DistributedArray.to_dist(np.zeros(nb)), niter=20, tol=0.0)
        x = solver.run(x, 10)
        assert solver.graph_error is None and solver.graph_replays > 0
        big = pm.MatrixMult(torch.ones((16 * GT_ROWS, 1024), dtype=torch.float64, device="cuda"))   # 32x the partials
        assert torch.all(big.rmatvec(torch.ones(16 * GT_ROWS, dtype=torch.float64, device="cuda")) == 16 * GT_ROWS)
        x = solver.run(x, 20)
        assert solver.graph_error is None and solver.graph_replays > 0
        assert solver.iiter == 20
        got = x.asarray().cpu().numpy()
    mv = lambda a: o.SimArray(o.blockdiag([[A]], a.locs))                  # noqa: E731
    rmv = lambda a: o.SimArray(o.blockdiag([[A]], a.locs, adjoint=True))   # noqa: E731
    xo, *_ = o.cgls(mv, rmv, mv(o.SimArray([xt])), o.SimArray([np.zeros(nb)]), niter=20, tol=0.0)
    np.testing.assert_allclose(got, xo.asarray(), rtol=1e-9, atol=1e-12)


# ------------------------------------------------------------------------------------------------------------------
# j. operators on the shapes the launchers used to refuse (one rank)
# ------------------------------------------------------------------------------------------------------------------
def np_wide(a):
    return a.astype(np.complex128 if np.iscomplexobj(a) else np.float64)


def np_ints(rng, shape, dtype, lo=-1, hi=1):
    a = rng.integers(lo, hi + 1, shape).astype(np.float64)
    if np.dtype(dtype).kind == "c":
        a = a + 1j * rng.integers(lo, hi + 1, shape)
    return a.astype(dtype)


WIDE_BLOCKS = [("complex128", 3, 130_001), ("float32", 2, 520_001)]


@pytest.mark.parametrize("dtype,m,n", WIDE_BLOCKS)
def test_matrixmult_wide_block(pm, dtype, m, n):
    from pylops_mpi_b200.utils.dottest import dottest
    rng = np.random.default_rng(m + n)
    A = np_ints(rng, (m, n), dtype)
    blk = pm.MatrixMult(A)
    x, v = np_ints(rng, n, dtype, -3, 3), np_ints(rng, m, dtype, -3, 3)
    assert np.array_equal(blk.matvec(torch.as_tensor(x).cuda()).cpu().numpy(), np_wide(A) @ np_wide(x))
    assert np.array_equal(blk.rmatvec(torch.as_tensor(v).cuda()).cpu().numpy(), np_wide(A).conj().T @ np_wide(v))
    Op = pm.MPIBlockDiag([blk])
    u = pm.DistributedArray.to_dist(rng.standard_normal(n).astype(dtype))
    w = pm.DistributedArray.to_dist(rng.standard_normal(m).astype(dtype))
    # float32: sums of 520,001 rounded terms on both sides of the identity
    dottest(Op, u, w, rtol=1e-3 if dtype == "float32" else 1e-10)


@pytest.mark.parametrize("dtype,m,n", WIDE_BLOCKS)
def test_blockdiag_vstack_adjoint_wide_block(pm, dtype, m, n):
    rng = np.random.default_rng(m * n)
    A = np_ints(rng, (m, n), dtype)
    v = np_ints(rng, m, dtype, -3, 3)
    ref = np_wide(A).conj().T @ np_wide(v)
    for Op in (pm.MPIBlockDiag([pm.MatrixMult(A)]), pm.MPIVStack([pm.MatrixMult(A)])):
        got = Op.rmatvec(pm.DistributedArray.to_dist(v)).asarray().cpu().numpy()
        assert np.array_equal(got, ref), type(Op).__name__


@pytest.mark.parametrize("kind", ["block", "summa"])
@pytest.mark.parametrize("dtype,N,K", [("complex128", 3, 130_001), ("float32", 2, 520_001)])
def test_mpimatrixmult_single_column_wide_tile(pm, kind, dtype, N, K):
    """M = 1: the adjoint's tile product is b2_gemv with op H on the N x K tile (block without saveAt, and SUMMA)"""
    rng = np.random.default_rng(N + K)
    A = np_ints(rng, (N, K), dtype)
    Op = pm.MPIMatrixMult(A, 1, kind=kind, dtype=dtype)
    x, v = np_ints(rng, K, dtype, -3, 3), np_ints(rng, N, dtype, -3, 3)
    fwd = (Op @ pm.DistributedArray.to_dist(x)).asarray().cpu().numpy()
    adj = Op.rmatvec(pm.DistributedArray.to_dist(v)).asarray().cpu().numpy()
    assert np.array_equal(fwd, np_wide(A) @ np_wide(x))
    assert np.array_equal(adj, np_wide(A).conj().T @ np_wide(v))


@pytest.mark.parametrize("kind", ["block", "summa"])
@pytest.mark.parametrize("N,K", [(GEMM_ROWS + 61, 2), (2, GEMM_ROWS + 61)])
def test_mpimatrixmult_tall_f32_three_columns(pm, kind, N, K):
    """M = 3, float32: the tile product is b2_gemm; N rows (forward) or K rows (adjoint) past 65535 row tiles"""
    rng = np.random.default_rng(N + 3 * K)
    M = 3
    A = np_ints(rng, (N, K), np.float32)
    Op = pm.MPIMatrixMult(A, M, kind=kind, dtype="float32")
    X, Y = np_ints(rng, (K, M), np.float32, -3, 3), np_ints(rng, (N, M), np.float32, -3, 3)
    fwd = (Op @ pm.DistributedArray.to_dist(X.ravel())).asarray().cpu().numpy()
    adj = Op.rmatvec(pm.DistributedArray.to_dist(Y.ravel())).asarray().cpu().numpy()
    A64 = A.astype(np.float64)
    assert np.array_equal(fwd, (A64 @ X).ravel())
    assert np.array_equal(adj, (A64.T @ Y).ravel())
