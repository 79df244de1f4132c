"""Derivative stencils (csrc/stencil.cu) against exact references.

Every per-rank entry point is called through the C ABI for each simulated rank of a row split, with its halo
rows taken from the same global device array, so one output array holds the whole operator's result.

* Applied to ``X = [I_N | 0]`` with sampling 1 the kernels return the operator's matrix: every output element
  is one tap times 1.0, so it is compared BIT FOR BIT with the dense oracle matrices (and their transposes for
  the adjoint), for every kind / order / edge, every small N, f32 and f64, the 16-byte vector kernel and the
  generic one, and row splits with 1-row ranks next to the global edges.
* The halo contract: a call is refused with B2_ERR_HALO exactly when it is given fewer halo rows than the taps of
  its rows read, and an accepted call gives the same rows as with the full halo.
* Random data: element-wise rounding bounds against a high-precision reference, and bitwise invariance of the
  result under the row split and the kernel variant (vector vs generic).
* The grid.y chunking of ``b2_derivative_axis`` and the multi-chunk pipeline of ``b2_first_derivative_host``.
* The row split of the overlapped halo exchange in ``MPIFirstDerivative._apply`` (``halo_launches``).
"""
import ctypes as C

import numpy as np
import pytest
import torch

import pylops_mpi_oracle as o
from pylops_mpi_b200.utils.partition import halo_launches, halo_plan, local_split_sizes, offsets

KINDS = {"forward": 0, "backward": 1, "centered": 2}
B2_OK, B2_ERR_DTYPE, B2_ERR_ARG, B2_ERR_HALO = 0, 2001, 2002, 2003
B2_ERR_WORKSPACE, B2_ERR_UNSUPPORTED, B2_ERR_ALIGN = 2004, 2005, 2006
# (deriv, kind, order, edge): every operator the stencil kernels apply
OPS = ([(1, k, order, e) for k, order in (("forward", 3), ("backward", 3), ("centered", 3), ("centered", 5))
        for e in (False, True)] + [(2, k, 3, e) for k in KINDS for e in (False, True)])
TORCH_DT = {"f32": torch.float32, "f64": torch.float64}
EPS = {torch.float32: float(np.finfo(np.float32).eps), torch.float64: float(np.finfo(np.float64).eps)}
NTAPS = 5


@pytest.fixture(scope="module")
def L():
    import pylops_mpi_b200._lib as L
    return L


def opname(op, adjoint=None):
    deriv, kind, order, edge = op
    s = f"d{deriv} {kind}{order if deriv == 1 else ''} edge={edge}"
    return s if adjoint is None else f"{s} adj={adjoint}"


_REACH = {}


def reach(L, op, adjoint):
    """(rows below, rows above) the stencil reads, as the library reports it"""
    key = (op, bool(adjoint))
    if key not in _REACH:
        deriv, kind, order, edge = op
        lo, hi = C.c_int(), C.c_int()
        if deriv == 1:
            L.check(L.lib.b2_first_derivative_halo(KINDS[kind], order, int(adjoint), C.byref(lo), C.byref(hi)))
        else:
            L.check(L.lib.b2_second_derivative_halo(KINDS[kind], int(edge), int(adjoint), C.byref(lo), C.byref(hi)))
        _REACH[key] = (lo.value, hi.value)
    return _REACH[key]


def block_reads(M, r0, r1):
    """(rows below, rows above) the block [r0, r1) reads: the non-zeros of its rows of the operator matrix M"""
    cols = np.nonzero(M[r0:r1])[1]
    if cols.size == 0:
        return 0, 0
    return max(0, r0 - int(cols.min())), max(0, int(cols.max()) - (r1 - 1))


def dense(op, N, h=1.0):
    """the oracle's N x N matrix, or None where it cannot be built (N too small for the edge stencil)"""
    deriv, kind, order, edge = op
    try:
        if deriv == 1:
            return o.first_derivative_dense(N, h, kind, edge, order)
        return o.second_derivative_dense(N, h, kind, edge)
    except IndexError:
        return None


def call(L, op, X, Y, N, r0, r1, n_lo, n_hi, h, adjoint, ctx=None, stream=None):
    """rows [r0, r1) of the global N-row array X (device, C order) -> the same rows of Y, as one rank of a split
    whose n_lo / n_hi halo rows are the rows of X around the block; returns the status code"""
    deriv, kind, order, edge = op
    ncols = X.numel() // N
    row = ncols * X.element_size()
    xb, yb = X.data_ptr(), Y.data_ptr()
    code = L.F32 if X.dtype is torch.float32 else L.F64
    args = (ctx or L.ctx(), xb + r0 * row, yb + r0 * row, xb + (r0 - n_lo) * row if n_lo else None, n_lo,
            xb + r1 * row if n_hi else None, n_hi, r1 - r0, ncols, r0, N)
    st = L.stream() if stream is None else stream
    if deriv == 1:
        return L.lib.b2_first_derivative(*args, KINDS[kind], order, int(edge), float(h), int(adjoint), code, st)
    return L.lib.b2_second_derivative(*args, KINDS[kind], int(edge), float(h), int(adjoint), code, st)


def full_halo(L, op, adjoint, N, r0, r1):
    nl, nh = reach(L, op, adjoint)
    return min(nl, r0), min(nh, N - r1)


def apply_split(L, op, X, Y, N, rows, h, adjoint):
    off = offsets(rows)
    for q in range(len(rows)):
        r0, r1 = off[q], off[q + 1]
        n_lo, n_hi = full_halo(L, op, adjoint, N, r0, r1)
        rc = call(L, op, X, Y, N, r0, r1, n_lo, n_hi, h, adjoint)
        assert rc == 0, f"{opname(op, adjoint)} N={N} split={rows} rank {q}: status {rc}"


def splits(N, pmax=4, all_ones_upto=8):
    """balanced splits over 1..pmax ranks, 1-row ranks at either / both global edges, all-1-row splits"""
    out = {tuple(local_split_sizes(N, P)) for P in range(1, min(pmax, N) + 1)}
    if N >= 2:
        out |= {(1, N - 1), (N - 1, 1)}
    if N >= 3:
        out.add((1, N - 2, 1))
    if N >= 5:
        out |= {(1, 1, N - 3, 1), (1, N - 3, 1, 1), (2, N - 3, 1)}
    if N <= all_ones_upto:
        out.add((1,) * N)
    return sorted(out, key=lambda s: (len(s), s))


def device_array(shape, dt, aligned, fill=0.0):
    """device array whose base is 16-byte aligned (vector kernel eligible when the rows are too) or one element
    past it (the generic kernel); a stack of [N x ncols] arrays keeps that property in every slice"""
    n = int(np.prod(shape))
    buf = torch.full((n + 1,), fill, dtype=dt, device="cuda")
    return (buf[:n] if aligned else buf[1:]).view(*shape)


def band_apply(M, x):
    """M @ x in long double for a matrix with non-zeros on diagonals -2..2 only (checked)"""
    N = M.shape[0]
    assert not np.triu(M, 3).any() and not np.tril(M, -3).any()
    y = np.zeros(x.shape, np.longdouble)
    for k in range(-2, 3):
        d = np.diagonal(M, k).astype(np.longdouble)[:, None]
        if k >= 0:
            y[:N - k] += d * x[k:]
        else:
            y[-k:] += d * x[:N + k]
    return y


def vec_cols(N, dt):
    V = 16 // torch.empty((), dtype=dt).element_size()
    return max(-(-N // V) * V, 8 * V)


# --------------------------------------------------------------------------
# (a) + (b): the operator matrix, bit for bit, and the halo contract
# --------------------------------------------------------------------------
NS = list(range(1, 25)) + [31, 32, 33, 63, 64, 65]


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["vec", "generic"])
@pytest.mark.parametrize("dt", ["f32", "f64"])
@pytest.mark.parametrize("N", NS)
def test_operator_matrix_exact(L, N, dt, layout):
    tdt = TORCH_DT[dt]
    npdt = np.float32 if dt == "f32" else np.float64
    ncols = vec_cols(N, tdt)
    vec = layout == "vec"
    X = device_array((N, ncols), tdt, vec)
    X[:, :N] = torch.eye(N, dtype=tdt, device="cuda")
    S = splits(N)
    blocks = [(s, rows, q, o0, o1) for s, rows in enumerate(S)
              for q, (o0, o1) in enumerate(zip(offsets(rows)[:-1], offsets(rows)[1:]))]
    for op in OPS:
        mats = {}
        for adjoint in (False, True):
            name = f"{opname(op, adjoint)} N={N} {dt} {layout}"
            Ys = device_array((len(S), N, ncols), tdt, vec, float("nan"))
            for s, rows in enumerate(S):
                apply_split(L, op, X, Ys[s], N, list(rows), 1.0, adjoint)
            # (b): every block again with fewer halo rows on one side: refused exactly when the taps of its rows
            # read a missing row (the non-zeros of the oracle matrix, sampling 1); where the oracle cannot build the
            # matrix, B2_ERR_HALO or the same rows
            D = dense(op, N)
            M = None if D is None else (D.T if adjoint else D)
            cuts = []
            for s, rows, q, r0, r1 in blocks:
                n_lo, n_hi = full_halo(L, op, adjoint, N, r0, r1)
                cuts += [(s, rows, q, r0, r1, a, n_hi, n_lo, n_hi) for a in range(n_lo)]
                cuts += [(s, rows, q, r0, r1, n_lo, b, n_lo, n_hi) for b in range(n_hi)]
            Zs = device_array((max(len(cuts), 1), N, ncols), tdt, vec, float("nan"))
            short = []
            for k, (s, rows, q, r0, r1, a, b, n_lo, n_hi) in enumerate(cuts):
                rc = call(L, op, X, Zs[k], N, r0, r1, a, b, 1.0, adjoint)
                if M is None:
                    assert rc in (0, B2_ERR_HALO), f"{name} split={rows} rank {q} halo ({a},{b}): status {rc}"
                else:
                    rl, rh = block_reads(M, r0, r1)
                    want = B2_ERR_HALO if a < rl or b < rh else 0
                    assert rc == want, (f"{name} split={rows} rank {q} (rows {r0}:{r1}) reads ({rl},{rh}), given "
                                        f"({a},{b}) halo rows: status {rc}, want {want}")
                if rc == 0:
                    short.append((k, s, rows, q, r0, r1, a, b, n_lo, n_hi))
            got = Ys.cpu().numpy()
            for s, rows in enumerate(S):
                assert np.array_equal(got[s][:, N:], np.zeros((N, ncols - N), npdt)), f"{name} split={rows}: pad"
                assert np.array_equal(got[s], got[0]), f"{name}: split {rows} differs from {S[0]}"
            zs = Zs.cpu().numpy()
            for k, s, rows, q, r0, r1, a, b, n_lo, n_hi in short:
                z = zs[k][r0:r1]
                assert np.array_equal(z, got[s][r0:r1]), (
                    f"{name} split={rows} rank {q} (rows {r0}:{r1}): {a} lo / {b} hi halo rows instead of "
                    f"{n_lo} / {n_hi} returned B2_OK with a different result")
            mats[adjoint] = got[0][:, :N]
            if M is not None:
                ref = M.astype(npdt)
                bad = np.argwhere(mats[adjoint] != ref)
                assert bad.size == 0, (f"{name}: matrix differs from the oracle at {bad[:4].tolist()}: "
                                       f"got {mats[adjoint][tuple(bad[0])]}, want {ref[tuple(bad[0])]}")
        # where the oracle cannot build the matrix, the adjoint is still the exact transpose
        assert np.array_equal(mats[True], mats[False].T), f"{opname(op)} N={N} {dt} {layout}: adjoint != forward^T"


@pytest.mark.gpu
def test_second_derivative_short_halo_is_an_error(L):
    """centered second derivative with edges: global row 0 reads row 2, so its adjoint at row 2 reads row 0; a
    block that starts at row 2 with one lo halo row (or ends at row 1 with one hi halo row) cannot be applied"""
    X = device_array((8, 32), torch.float64, True, 1.0)
    Y = device_array((8, 32), torch.float64, True)
    op = (2, "centered", 3, True)
    assert call(L, op, X, Y, 8, 2, 8, 1, 0, 1.0, True) == B2_ERR_HALO
    assert call(L, op, X, Y, 8, 0, 1, 0, 1, 1.0, False) == B2_ERR_HALO
    assert call(L, op, X, Y, 8, 2, 8, 2, 0, 1.0, True) == 0
    assert call(L, op, X, Y, 8, 3, 8, 1, 0, 1.0, True) == 0      # row 3 and above read one row below
    op = (2, "centered", 3, False)
    assert call(L, op, X, Y, 8, 2, 8, 1, 0, 1.0, True) == 0
    assert call(L, op, X, Y, 8, 2, 8, 0, 0, 1.0, True) == B2_ERR_HALO


# (op, adjoint, block [r0, r1) of N = 8 rows, lo / hi halo rows given, status)
SHORT_HALO_CASES = {
    "d1_centered3_rows0to1_hi_0": ((1, "centered", 3, False), False, 0, 1, 0, 0, B2_OK),
    "d1_centered3_adj_rows0to1_hi_0": ((1, "centered", 3, False), True, 0, 1, 0, 0, B2_ERR_HALO),
    "d1_centered3_edge_rows0to1_hi_0": ((1, "centered", 3, True), False, 0, 1, 0, 0, B2_ERR_HALO),
    "d1_centered5_rows0to2_hi_0": ((1, "centered", 5, False), False, 0, 2, 0, 0, B2_OK),
    "d1_centered5_edge_rows0to1_hi_1": ((1, "centered", 5, True), False, 0, 1, 0, 1, B2_OK),
    "d1_centered5_edge_rows0to2_hi_1": ((1, "centered", 5, True), False, 0, 2, 0, 1, B2_OK),
    "d1_centered5_edge_rows0to3_hi_1": ((1, "centered", 5, True), False, 0, 3, 0, 1, B2_ERR_HALO),
    "d1_forward_rows3to4_hi_0": ((1, "forward", 3, False), False, 3, 4, 1, 0, B2_ERR_HALO),
    "d1_forward_adj_rows3to4_lo_0": ((1, "forward", 3, False), True, 3, 4, 0, 1, B2_ERR_HALO),
    "d1_forward_adj_rows3to4_hi_0": ((1, "forward", 3, False), True, 3, 4, 1, 0, B2_OK),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(SHORT_HALO_CASES))
def test_first_derivative_short_halo_cases(L, case):
    """first-derivative blocks given fewer halo rows than the operator's reach: refused exactly when their own rows
    read a missing row; an accepted block gives the rows of a full-halo call"""
    op, adjoint, r0, r1, n_lo, n_hi, want = SHORT_HALO_CASES[case]
    gen = torch.Generator(device="cuda").manual_seed(3)
    X = torch.randn(8, 32, dtype=torch.float64, device="cuda", generator=gen)
    Y = device_array((8, 32), torch.float64, True, float("nan"))
    Z = device_array((8, 32), torch.float64, True, float("nan"))
    assert call(L, op, X, Y, 8, r0, r1, n_lo, n_hi, 1.0, adjoint) == want
    if want == B2_OK:
        L.check(call(L, op, X, Z, 8, r0, r1, *full_halo(L, op, adjoint, 8, r0, r1), 1.0, adjoint))
        assert torch.equal(Y[r0:r1], Z[r0:r1])


def test_halo_reach_values(L):
    """the rows below / above itself that any row of each stencil reads, (forward operator, adjoint)"""
    first = {("forward", 3): ((0, 1), (1, 0)), ("backward", 3): ((1, 0), (0, 1)),
             ("centered", 3): ((1, 1), (1, 1)), ("centered", 5): ((2, 2), (2, 2))}
    second = {("forward", False): ((0, 2), (2, 0)), ("forward", True): ((0, 2), (2, 0)),
              ("backward", False): ((2, 0), (0, 2)), ("backward", True): ((2, 0), (0, 2)),
              ("centered", False): ((1, 1), (1, 1)), ("centered", True): ((2, 2), (2, 2))}

    def halo(fn, *args):
        lo, hi = C.c_int(-1), C.c_int(-1)
        return fn(*args, C.byref(lo), C.byref(hi)), (lo.value, hi.value)

    for (kind, order), want in first.items():
        for adjoint in (0, 1):
            assert halo(L.lib.b2_first_derivative_halo, KINDS[kind], order, adjoint) == (B2_OK, want[adjoint]), \
                f"d1 {kind}{order} adj={adjoint}"
    for (kind, edge), want in second.items():
        for adjoint in (0, 1):
            assert halo(L.lib.b2_second_derivative_halo, KINDS[kind], int(edge), adjoint) == (B2_OK, want[adjoint]), \
                f"d2 {kind} edge={edge} adj={adjoint}"
    assert L.lib.b2_first_derivative_halo(KINDS["centered"], 5, 0, None, None) == B2_OK
    assert L.lib.b2_second_derivative_halo(KINDS["centered"], 1, 1, None, None) == B2_OK
    for bad in (-1, 3):
        assert halo(L.lib.b2_first_derivative_halo, bad, 3, 0)[0] == B2_ERR_UNSUPPORTED
        assert halo(L.lib.b2_second_derivative_halo, bad, 0, 0)[0] == B2_ERR_UNSUPPORTED
    for adjoint in (0, 1):
        assert halo(L.lib.b2_first_derivative_halo, KINDS["centered"], 4, adjoint)[0] == B2_ERR_UNSUPPORTED


# the argument checks of the five entry points that run the stencil kernels: every row changes one or two arguments
# of a valid call (a None entry passes NULL) and gives the status; rows that pass every check launch on valid memory
FD = dict(ctx=1, x=1, y=1, lo=None, n_lo=0, hi=None, n_hi=0, nloc=8, ncols=32, row0=0, nglob=8, kind=2, order=3,
          edge=0, h=1.0, adj=0, dtype=1)
FD_ARGS = [
    ({}, B2_OK), ({"ctx": None}, B2_ERR_ARG), ({"ctx": None, "nloc": 0}, B2_ERR_ARG),
    ({"nloc": 0, "x": None}, B2_OK), ({"ncols": 0, "y": None}, B2_OK), ({"x": None}, B2_ERR_ARG),
    ({"y": None}, B2_ERR_ARG), ({"n_lo": -1}, B2_ERR_ARG), ({"n_hi": -1}, B2_ERR_ARG),
    ({"lo": 1, "n_lo": 9}, B2_ERR_ARG), ({"hi": 1, "n_hi": 9}, B2_ERR_ARG), ({"n_lo": 9}, B2_ERR_ARG),
    ({"kind": 3}, B2_ERR_UNSUPPORTED), ({"kind": -1}, B2_ERR_UNSUPPORTED), ({"kind": 3, "nloc": 0}, B2_OK),
    ({"kind": 3, "dtype": 3}, B2_ERR_UNSUPPORTED), ({"dtype": 3}, B2_ERR_DTYPE), ({"dtype": 99}, B2_ERR_DTYPE),
    ({"dtype": 99, "nloc": 0}, B2_OK), ({"row0": 4, "nloc": 8, "lo": 1, "n_lo": 1}, B2_ERR_ARG),
]
FD1_ARGS = FD_ARGS + [({"order": 4}, B2_ERR_UNSUPPORTED), ({"order": 4, "kind": 0}, B2_OK),
                      ({"order": 4, "dtype": 3}, B2_ERR_UNSUPPORTED)]
AX = dict(ctx=1, x=1, y=1, n_outer=1, n_axis=8, n_inner=32, deriv=1, kind=2, order=3, edge=0, h=1.0, adj=0, dtype=1)
AX_ARGS = [
    ({}, B2_OK), ({"deriv": 2}, B2_OK), ({"ctx": None}, B2_ERR_ARG), ({"deriv": 0}, B2_ERR_ARG),
    ({"deriv": 3}, B2_ERR_ARG), ({"deriv": 0, "n_outer": 0}, B2_ERR_ARG), ({"n_outer": 0, "x": None}, B2_OK),
    ({"n_axis": 0}, B2_OK), ({"n_inner": 0}, B2_OK), ({"x": None}, B2_ERR_ARG), ({"y": None}, B2_ERR_ARG),
    ({"kind": 3}, B2_ERR_UNSUPPORTED), ({"kind": 3, "n_inner": 0}, B2_OK), ({"order": 4}, B2_ERR_UNSUPPORTED),
    ({"order": 4, "deriv": 2}, B2_OK), ({"kind": 3, "dtype": 99}, B2_ERR_UNSUPPORTED), ({"dtype": 3}, B2_ERR_DTYPE),
    ({"dtype": 99}, B2_ERR_DTYPE),
]
# the handle's boxes hold one 32-column float64 row per side: every row here fails before the launch
PEER = dict(ctx=1, h=1, x=1, y=1, nloc=8, ncols=32, row0=0, nglob=8, deriv=1, kind=2, order=3, edge=0, sh=1.0, adj=0,
            dtype=1)
PEER_ARGS = [
    ({"row0": 4}, B2_ERR_ARG), ({"ctx": None}, B2_ERR_ARG), ({"h": None}, B2_ERR_ARG), ({"x": None}, B2_ERR_ARG),
    ({"y": None}, B2_ERR_ARG), ({"deriv": 0}, B2_ERR_ARG), ({"deriv": 3}, B2_ERR_ARG),
    ({"deriv": 0, "dtype": 3}, B2_ERR_ARG), ({"dtype": 3}, B2_ERR_DTYPE), ({"dtype": 3, "kind": 3}, B2_ERR_DTYPE),
    ({"kind": 3}, B2_ERR_UNSUPPORTED), ({"kind": -1, "nloc": 0}, B2_ERR_UNSUPPORTED),
    ({"order": 4}, B2_ERR_UNSUPPORTED), ({"order": 4, "deriv": 2, "row0": 4}, B2_ERR_ARG),
    ({"nloc": 0}, B2_ERR_HALO), ({"order": 5, "nloc": 1}, B2_ERR_HALO),
    ({"deriv": 2, "edge": 1, "nloc": 1}, B2_ERR_HALO),
    ({"ncols": 31}, B2_ERR_ALIGN), ({"ncols": 14}, B2_ERR_ALIGN), ({"x": 8}, B2_ERR_ALIGN),
    ({"order": 5}, B2_ERR_WORKSPACE), ({"deriv": 2, "kind": 0}, B2_ERR_WORKSPACE),
]
HOST = dict(ctx=1, x=1, y=1, nglob=8, ncols=32, begin=0, end=8, kind=2, order=3, edge=0, h=1.0, adj=0, dtype=1)
HOST_ARGS = [
    ({}, B2_OK), ({"ctx": None}, B2_ERR_ARG), ({"end": 9}, B2_ERR_ARG), ({"begin": 5, "end": 4}, B2_ERR_ARG),
    ({"begin": 4, "end": 4, "x": None}, B2_OK), ({"ncols": 0, "y": None}, B2_OK), ({"x": None}, B2_ERR_ARG),
    ({"y": None}, B2_ERR_ARG), ({"dtype": 3}, B2_ERR_DTYPE), ({"dtype": 3, "kind": 3}, B2_ERR_DTYPE),
    ({"kind": 3}, B2_ERR_UNSUPPORTED), ({"order": 4}, B2_ERR_UNSUPPORTED), ({"order": 4, "kind": 1}, B2_OK),
]


@pytest.mark.gpu
def test_entry_point_argument_errors(L):
    X = device_array((8, 32), torch.float64, True, 1.0)
    Y = device_array((8, 32), torch.float64, True)
    ptr = {"x": X.data_ptr(), "y": Y.data_ptr(), "lo": X.data_ptr(), "hi": X.data_ptr()}
    st = L.stream()

    def args(base, change, fields):
        a = dict(base, **change)
        out = []
        for f in fields:
            v = a[f]
            if f == "ctx":
                v = L.ctx() if v else None
            elif f in ptr and v is not None:
                v = ptr[f] + (v if v > 1 else 0)          # an int > 1 is a byte offset
            out.append(v)
        return out

    fd = ["ctx", "x", "y", "lo", "n_lo", "hi", "n_hi", "nloc", "ncols", "row0", "nglob", "kind"]
    bad = []
    for change, want in FD1_ARGS:
        rc = L.lib.b2_first_derivative(*args(FD, change, fd + ["order", "edge", "h", "adj", "dtype"]), st)
        if rc != want:
            bad.append(("b2_first_derivative", change, rc, want))
    for change, want in FD_ARGS:
        rc = L.lib.b2_second_derivative(*args(FD, change, fd + ["edge", "h", "adj", "dtype"]), st)
        if rc != want:
            bad.append(("b2_second_derivative", change, rc, want))
    for change, want in AX_ARGS:
        rc = L.lib.b2_derivative_axis(*args(AX, change, ["ctx", "x", "y", "n_outer", "n_axis", "n_inner", "deriv",
                                                         "kind", "order", "edge", "h", "adj", "dtype"]), st)
        if rc != want:
            bad.append(("b2_derivative_axis", change, rc, want))
    cap = 32 * 8
    box = torch.zeros(L.lib.b2_mailbox_bytes(cap), dtype=torch.uint8, device="cuda")
    boxes = (C.c_void_p * 1)(box.data_ptr())
    h = C.c_void_p()
    L.check(L.lib.b2_mailbox_create(0, 1, boxes, cap, C.byref(h)), "b2_mailbox_create")
    try:
        for change, want in PEER_ARGS:
            a = args(PEER, change, ["ctx", "h", "x", "y", "nloc", "ncols", "row0", "nglob", "deriv", "kind", "order",
                                    "edge", "sh", "adj", "dtype"])
            a[1] = h if a[1] else None
            rc = L.lib.b2_derivative_peer(*a, st)
            if rc != want:
                bad.append(("b2_derivative_peer", change, rc, want))
    finally:
        L.check(L.lib.b2_mailbox_destroy(h), "b2_mailbox_destroy")
    xh, yh = np.ones((8, 32)), np.zeros((8, 32))
    ptr.update(x=xh.ctypes.data, y=yh.ctypes.data)
    for change, want in HOST_ARGS:
        rc = L.lib.b2_first_derivative_host(*args(HOST, change, ["ctx", "x", "y", "nglob", "ncols", "begin", "end",
                                                                 "kind", "order", "edge", "h", "adj", "dtype"]))
        if rc != want:
            bad.append(("b2_first_derivative_host", change, rc, want))
    torch.cuda.synchronize()
    assert not bad, "\n".join(f"{fn} {change}: status {rc}, want {want}" for fn, change, rc, want in bad)


# --------------------------------------------------------------------------
# (c) random data, sampling != 1, complex as twice-wide real rows: element-wise rounding bound
# --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["f32", "f64", "c64", "c128"])
@pytest.mark.parametrize("N", [5, 9, 37, 130])
def test_random_rounding_bound(L, N, dt):
    cplx = dt in ("c64", "c128")
    tdt = torch.float32 if dt in ("f32", "c64") else torch.float64
    rng = np.random.default_rng(N)
    m = 40 if cplx else 80                                     # complex: m values = 2m real columns
    x = rng.standard_normal((N, m)) * 10 ** rng.uniform(-3, 3, (N, 1))
    if cplx:
        x = x + 1j * rng.standard_normal((N, m))
        xr = x.astype(np.complex64 if dt == "c64" else np.complex128).view(
            np.float32 if dt == "c64" else np.float64)
    else:
        xr = x.astype(np.float32 if dt == "f32" else np.float64)
    X = torch.as_tensor(xr).cuda()
    xl = xr.astype(np.longdouble)
    eps = EPS[tdt]
    for op in OPS:
        D0 = dense(op, N)
        for adjoint in (False, True):
            M = D0.T if adjoint else D0
            ref0 = band_apply(M, xl)
            bound0 = (NTAPS + 1) * eps * (np.abs(M) @ np.abs(xr.astype(np.float64)))
            for h in (0.37, 3.0):
                scale = 1.0 / h if op[0] == 1 else 1.0 / (h * h)
                ref = ref0 / (np.longdouble(h) if op[0] == 1 else np.longdouble(h) * np.longdouble(h))
                bound = bound0 * scale
                for rows in (local_split_sizes(N, 1), local_split_sizes(N, 3), [1, N - 2, 1]):
                    Y = torch.full_like(X, float("nan"))
                    apply_split(L, op, X, Y, N, rows, h, adjoint)
                    err = np.abs(Y.cpu().numpy().astype(np.longdouble) - ref).astype(np.float64)
                    bad = np.argwhere(~(err <= bound))
                    assert bad.size == 0, (f"{opname(op, adjoint)} N={N} {dt} h={h} split={rows}: error "
                                           f"{err[tuple(bad[0])]:.3e} > bound {bound[tuple(bad[0])]:.3e} at "
                                           f"{bad[0].tolist()}")


# --------------------------------------------------------------------------
# (d) bitwise invariances: row split, vector vs generic kernel
# --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["f32", "f64"])
@pytest.mark.parametrize("N,nvec", [(37, 8), (66, 8), (37, 130), (13, 9)])
def test_split_and_kernel_invariance(L, N, nvec, dt):
    """nloc not a multiple of the 4-row chunk, exactly 8 column vectors (the smallest vector launch), 130 vectors
    (a partial 128-wide column tile): every split and both kernels give the same bits"""
    tdt = TORCH_DT[dt]
    ncols = nvec * (16 // torch.empty((), dtype=tdt).element_size())
    gen = torch.Generator(device="cuda").manual_seed(N * 1000 + nvec)
    src = torch.randn(N, ncols, dtype=tdt, device="cuda", generator=gen)
    Xs = {}
    for layout in ("vec", "generic"):
        Xs[layout] = device_array((N, ncols), tdt, layout == "vec")
        Xs[layout].copy_(src)
    S = sorted({tuple(local_split_sizes(N, P)) for P in range(1, 7)} |
               {(1, N - 1), (N - 1, 1), (1, N - 2, 1), (1, 1, N - 4, 1, 1), (2, 1, N - 4, 1)}, key=len)
    for op in OPS:
        for adjoint in (False, True):
            base = None
            for layout, X in Xs.items():
                for rows in S:
                    Y = device_array((N, ncols), tdt, layout == "vec", float("nan"))
                    apply_split(L, op, X, Y, N, list(rows), 0.7, adjoint)
                    y = Y.cpu().numpy()
                    if base is None:
                        base = y
                        assert not np.isnan(base).any()
                    assert np.array_equal(y, base), f"{opname(op, adjoint)} N={N} {dt} {layout} split={rows}"


# --------------------------------------------------------------------------
# (e) b2_derivative_axis: more lines than one grid.y launch holds
# --------------------------------------------------------------------------
def axis_ref_check(name, y, x, D, eps):
    """y = D along axis 1 of x [n_outer, n_axis, n_inner], element-wise within the rounding bound"""
    x64 = x.astype(np.float64)
    ref = np.einsum("ij,ojk->oik", D, x64)
    bound = (NTAPS + 1) * eps * np.einsum("ij,ojk->oik", np.abs(D), np.abs(x64))
    err = np.abs(y.astype(np.float64) - ref)
    bad = np.argwhere(~(err <= bound + 1e-300))
    assert bad.size == 0, f"{name}: line {bad[0].tolist()} error {err[tuple(bad[0])]:.3e} > {bound[tuple(bad[0])]:.3e}"


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["f32", "f64"])
@pytest.mark.parametrize("layout", ["vec", "generic"])
@pytest.mark.parametrize("n_outer", [65535, 65536, 2 * 65535 + 7])
def test_derivative_axis_grid_chunks(L, n_outer, layout, dt):
    tdt = TORCH_DT[dt]
    code = L.F32 if dt == "f32" else L.F64
    n_inner = (32 if dt == "f32" else 16) if layout == "vec" else 1
    n_axis = 6 if n_outer < 2 * 65535 else 3          # <= ~50 MB per array
    gen = torch.Generator(device="cuda").manual_seed(n_outer + n_inner)
    X = torch.randn(n_outer, n_axis, n_inner, dtype=tdt, device="cuda", generator=gen)
    Y = torch.full_like(X, float("nan"))
    x = X.cpu().numpy()
    h = 0.8
    for deriv, kind, order, edge, adjoint in ((1, "centered", 5, True, False), (2, "centered", 3, True, True),
                                              (1, "forward", 3, False, True), (2, "backward", 3, False, False)):
        op = (deriv, kind, order, edge)
        L.check(L.lib.b2_derivative_axis(L.ctx(), X.data_ptr(), Y.data_ptr(), n_outer, n_axis, n_inner, deriv,
                                         KINDS[kind], order, int(edge), h, int(adjoint), code, L.stream()),
                "b2_derivative_axis")
        D = dense(op, n_axis, h)
        axis_ref_check(f"{opname(op, adjoint)} {n_outer}x{n_axis}x{n_inner} {dt}", Y.cpu().numpy(), x,
                       D.T if adjoint else D, EPS[tdt])


@pytest.mark.gpu
def test_local_first_derivative_last_axis_complex(L):
    """complex local.FirstDerivative along the last axis of a (300, 300, 9) block: 90000 lines of 9 samples"""
    from pylops_mpi_b200 import local
    dims = (300, 300, 9)
    rng = np.random.default_rng(5)
    x = rng.standard_normal(dims) + 1j * rng.standard_normal(dims)
    Op = local.FirstDerivative(dims, axis=-1, sampling=0.5, kind="centered", order=5, edge=True, dtype=np.complex128)
    D = o.first_derivative_dense(9, 0.5, "centered", True, 5)
    xd = torch.as_tensor(x.ravel()).cuda()
    for adjoint in (False, True):
        y = (Op.rmatvec(xd) if adjoint else Op.matvec(xd)).cpu().numpy().reshape(dims)
        xr = x.reshape(-1, 9, 1).view(np.float64).reshape(-1, 9, 2)
        yr = y.reshape(-1, 9, 1).view(np.float64).reshape(-1, 9, 2)
        axis_ref_check(f"local.FirstDerivative complex adj={adjoint}", yr, xr, D.T if adjoint else D, EPS[torch.float64])


# --------------------------------------------------------------------------
# (f) b2_first_derivative_host: several 64-row chunks over the three rotating streams
# --------------------------------------------------------------------------
@pytest.mark.gpu
def test_host_pipeline_multi_chunk(L):
    """512 KiB rows -> 64-row chunks; 389 rows = 7 chunks, so every stream slot and its buffers are reused.  A
    private context makes the first large call re-allocate the buffers a small call left behind.  The output is
    bit-identical to the device-resident kernel on the same rows and halos, and sampled columns match the dense
    operator within the rounding bound."""
    N = 6 * 64 + 5
    ctx = C.c_void_p()
    L.check(L.lib.b2_ctx_create(torch.cuda.current_device(), C.byref(ctx)), "b2_ctx_create")
    try:
        for dt, code in ((torch.float32, L.F32), (torch.float64, L.F64)):
            ncols = (512 << 10) // torch.empty((), dtype=dt).element_size()
            # small call first: the pipeline buffers are sized for it, then grown
            xs = torch.randn(8, 64, dtype=dt).pin_memory()
            ys = torch.empty_like(xs).pin_memory()
            L.check(L.lib.b2_first_derivative_host(ctx, xs.data_ptr(), ys.data_ptr(), 8, 64, 0, 8, 2, 3, 1, 1.0, 0,
                                                   code), "fd_host small")
            ref_s = o.first_derivative_dense(8, 1.0, "centered", True, 3) @ xs.numpy().astype(np.float64)
            np.testing.assert_allclose(ys.numpy(), ref_s, rtol=4 * EPS[dt], atol=4 * EPS[dt] * np.abs(ref_s).max())
            gen = torch.Generator(device="cuda").manual_seed(11)
            Xd = torch.randn(N, ncols, dtype=dt, device="cuda", generator=gen)
            xh = torch.empty((N, ncols), dtype=dt, pin_memory=True)
            xh.copy_(Xd)
            yh = torch.empty((N, ncols), dtype=dt, pin_memory=True)
            Yd = torch.empty_like(Xd)
            cols = np.arange(0, ncols, 4099)
            xc = xh.numpy()[:, cols].astype(np.float64)
            for (kind, order, edge, adjoint) in (("centered", 5, True, False), ("forward", 3, True, True)):
                op = (1, kind, order, edge)
                D = dense(op, N, 2.0)
                M = D.T if adjoint else D
                ref = M @ xc
                bound = (NTAPS + 1) * EPS[dt] * (np.abs(M) @ np.abs(xc))
                for b, e in ((0, N), (3, N - 70), (130, N)):
                    name = f"{opname(op, adjoint)} {dt} rows {b}:{e}"
                    yh.fill_(float("nan"))
                    L.check(L.lib.b2_first_derivative_host(ctx, xh.data_ptr(), yh.data_ptr(), N, ncols, b, e,
                                                           KINDS[kind], order, int(edge), 2.0, int(adjoint), code),
                            "fd_host " + name)
                    n_lo, n_hi = full_halo(L, op, adjoint, N, b, e)
                    L.check(call(L, op, Xd, Yd, N, b, e, n_lo, n_hi, 2.0, adjoint), "fd " + name)
                    assert torch.equal(yh[b:e], Yd[b:e].cpu()), f"{name}: host pipeline != device kernel"
                    assert torch.isnan(yh[:b]).all() and torch.isnan(yh[e:]).all(), f"{name}: wrote outside rows"
                    err = np.abs(yh.numpy()[b:e][:, cols].astype(np.float64) - ref[b:e])
                    assert (err <= bound[b:e]).all(), f"{name}: sampled columns outside the rounding bound"
            del xh, yh, Xd, Yd
    finally:
        L.check(L.lib.b2_ctx_destroy(ctx), "b2_ctx_destroy")


# --------------------------------------------------------------------------
# (g) the row split of the overlapped halo exchange (MPIFirstDerivative._apply)
# --------------------------------------------------------------------------
def test_halo_launches_invariants():
    """the launches tile the block; each is given the rows its stencil reads wherever those rows exist; launches
    that read received rows come after the exchange; with the full reach received (every balanced split) the
    interior launch is [n_lo, nloc - n_hi)"""
    for nloc in range(1, 31):
        for nl in range(3):
            for nh in range(3):
                for n_lo in range(nl + 1):
                    for n_hi in range(nh + 1):
                        case = f"nloc={nloc} reach=({nl},{nh}) received=({n_lo},{n_hi})"
                        steps = halo_launches(nloc, nl, nh, n_lo, n_hi)
                        spans = sorted((b, e) for b, e, *_ in steps)
                        bounds = [b for b, _ in spans] + [spans[-1][1]]
                        assert bounds[0] == 0 and bounds[-1] == nloc, case
                        assert all(spans[i][1] == spans[i + 1][0] for i in range(len(spans) - 1)), case
                        for b, e, lo, hi, after in steps:
                            assert b < e, case
                            if b == 0:
                                assert lo == n_lo, case
                            else:
                                assert lo <= b and lo >= min(nl, b + n_lo), f"{case}: launch [{b},{e}) lo={lo}"
                            if e == nloc:
                                assert hi == n_hi, case
                            else:
                                assert hi <= nloc - e and hi >= min(nh, nloc - e + n_hi), \
                                    f"{case}: launch [{b},{e}) hi={hi}"
                            reads_received = (b == 0 and lo > 0) or (e == nloc and hi > 0)
                            assert after or not reads_received, f"{case}: [{b},{e}) reads halo before the exchange"
                        if len(steps) > 1 or not steps[0][4]:
                            assert not steps[0][4] and all(s[4] for s in steps[1:]), case
                            if (n_lo, n_hi) == (nl, nh):
                                assert steps[0][:2] == (n_lo, nloc - n_hi), case


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["f32", "f64"])
@pytest.mark.parametrize("N", [12, 23])
def test_halo_launches_replay(L, N, dt):
    """replay every simulated rank's launch list (1-row blocks next to a global edge included) with the halo
    rows the exchange delivers: bit for bit the single-rank result"""
    tdt = TORCH_DT[dt]
    ncols = vec_cols(N, tdt)
    gen = torch.Generator(device="cuda").manual_seed(N)
    X = torch.randn(N, ncols, dtype=tdt, device="cuda", generator=gen)
    S = [local_split_sizes(N, P) for P in (2, 3, 4)] + [[1, N - 1], [N - 1, 1], [1, N - 2, 1], [1, 9, N - 10],
                                                        [N - 10, 9, 1], [2, N - 3, 1], [1, 1, N - 3, 1]]
    for op in OPS:
        for adjoint in (False, True):
            ref = torch.full_like(X, float("nan"))
            apply_split(L, op, X, ref, N, [N], 1.3, adjoint)
            nl, nh = reach(L, op, adjoint)
            for rows in S:
                off = offsets(rows)
                Y = torch.full_like(X, float("nan"))
                for q in range(len(rows)):
                    try:
                        plan = halo_plan(rows, q, nl, nh)
                    except ValueError:
                        break                       # the operator refuses this split as well
                    r0 = off[q]
                    for b, e, lo, hi, _ in halo_launches(rows[q], nl, nh, plan["recv_lo"], plan["recv_hi"]):
                        rc = call(L, op, X, Y, N, r0 + b, r0 + e, lo, hi, 1.3, adjoint)
                        assert rc == 0, (f"{opname(op, adjoint)} N={N} {dt} split={rows} rank {q}: launch "
                                         f"[{b},{e}) with {lo}/{hi} halo rows: status {rc}")
                else:
                    assert torch.equal(Y, ref), f"{opname(op, adjoint)} N={N} {dt} split={rows}"
