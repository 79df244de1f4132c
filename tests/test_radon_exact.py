"""The Radon and window kernels (b2_radon, b2_radon_windows, b2_radon_patches in csrc/radon.cu; b2_patch in
csrc/sliding.cu) against references that share no code with them, at the geometries they run in: curves that cross
the whole window, samples held by four windows along every axis, windows wider than one 256-term tile, grids past
the overlap-add kernel's block limit, and the benchmark's patch operators.

References (CPU, NumPy / SciPy, float64):

- ``radon_sparse``: the definition of test_radon.py (``tdec``, ``dense``) as a CSR matrix, vectorised over every
  (trace, model trace, t0);
- ``window_matrix``: the windowed operator  sum_w R_w^T diag(tap_w) A_w.  Window w = (i0, i1, i2) starts at
  (i0 step0, i1 step1, i2 step2) of the section [n0][n1][ns], the model blocks are window-major as local.py stores
  them, and tap_w is the taper in the data's type T: b2_radon_windows' T table, or b2_radon_patches'
  ((t0 * t1) * t2) formed in float64 and rounded once to T;
- ``emulate_forward`` / ``emulate_adjoint``: the order of operations that the header of csrc/radon.cu documents,
  evaluated at chosen outputs only.  Forward: each window's float64 sum over model traces in (py, px) order, t0
  ascending, rounded once to T, multiplied by the taper in T and added in T over i2 inside i1 inside i0.  Adjoint:
  per model sample a float64 sum over traces in (hy, hx) order of x[it] (1 - d) + x[it + 1] d, each x being tap * d
  rounded to T.  Sums are sequential (a loop over padded term columns), never np.sum, whose pairwise order differs.

The float64 bound of a windowed output (the kernel against the exact value of the definition):

    |got - M x| <= ((k + 3) u64 + (m + 2) u_T) (|M| |x|)

k is the largest number of terms in one window's float64 sum: each product w * x and each addition rounds once,
(k + 2) u64, plus one u64 for M's entries tap * w, which are themselves rounded products.  m is the largest number of
windows over one output sample (0 in the adjoint).  The T operations add u_T each: the rounding of the window sum to
T, the taper product, and up to m additions of the overlap sum (adjoint: the rounding of tap * d, and the final
rounding to T).  u_T is 2^-24 for float32 and 2^-53 for float64.  The reference M x is formed in extended precision,
so its own error is below k 2^-63 |M| |x|, which the bound also adds.  Every case asserts that the bound is not
vacuous: below 1e-12 of |M| |x| in float64, and below 1e-5 in float32.
"""
import copy
import itertools
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import test_patch  # noqa: E402
import test_sliding  # noqa: E402
from op_checks import guarded_twice, host  # noqa: E402
from test_radon import KERNEL_SHAPES, dense, kernel_axes, unitless  # noqa: E402

KINDS = ["linear", "parabolic", "hyperbolic"]
U64, U32, ULD = 2.0 ** -53, 2.0 ** -24, 2.0 ** -63
SPIKE = -0.7310585786300049          # a spike value with a full mantissa (rounded to T before use), not 1


def unit(dt):
    return U32 if dt == np.float32 else U64


# ---------------------------------------------------------------------------------------------------------------
# geometry
# ---------------------------------------------------------------------------------------------------------------
class Geo:
    """One call's geometry.  The Radon of one window: ``kind``, ``interp`` and the unitless axes ``hy``, ``hx``,
    ``py``, ``px`` (``hy = py = None`` in 2-D).  A window holds ``L = (nhy, nhx, nt)`` traces and samples, its model
    ``P = (npy, npx)`` traces of nt samples.  The section ``n = (n0, n1, ns)`` holds ``nw`` windows every ``st``.
    ``taper``: None, ``("table", tab)`` with tab ``[nw0 * nw1][nhy][nhx]`` float64 (b2_radon_windows rounds it to
    T), or ``("axis", [t0, t1, t2])`` float64 per-axis tables ``[nw_a][L_a]``, None where an axis is not tapered
    (b2_radon_patches).  ``entry`` is the C entry point: "radon" (one window, the whole section), "windows" or
    "patches"."""

    def __init__(self, entry, kind, interp, hy, hx, py, px, nt, n=None, nw=(1, 1, 1), st=(1, 1, 1), taper=None):
        self.entry, self.kind, self.interp = entry, kind, bool(interp)
        f = (lambda a: None if a is None else np.asarray(a, dtype=np.float64))
        self.hy, self.hx, self.py, self.px = f(hy), f(hx), f(py), f(px)
        self.L = (1 if hy is None else len(hy), len(hx), int(nt))
        self.P = (1 if py is None else len(py), len(px))
        self.n = self.L if n is None else tuple(int(v) for v in n)
        self.nw, self.st, self.taper = tuple(nw), tuple(st), taper
        self.nwin = int(np.prod(self.nw))
        self.nm = self.P[0] * self.P[1] * self.L[2]          # model values per window (one component)
        self.nd = int(np.prod(self.n))                        # section values (one component)

    def windows(self):
        return itertools.product(*[range(v) for v in self.nw])

    def covering(self, axis, a):
        """the windows along ``axis`` that hold index a, ascending"""
        return [i for i in range(self.nw[axis]) if i * self.st[axis] <= a < i * self.st[axis] + self.L[axis]]

    def depth(self):
        """the most windows over one section sample"""
        return int(np.prod([max(len(self.covering(ax, a)) for a in range(self.n[ax])) for ax in range(3)]))


def tap_window(G, dt, i0, i1, i2):
    """window (i0, i1, i2)'s taper at every window sample [nhy][nhx][nt], the values of T as float64"""
    if G.taper is None:
        return np.ones(G.L)
    how, t = G.taper
    if how == "table":
        tab = np.asarray(t[i0 * G.nw[1] + i1], dtype=dt).astype(np.float64)
        return np.broadcast_to(tab[:, :, None], G.L)
    a, b, c = (np.ones(G.L[ax]) if t[ax] is None else t[ax][i] for ax, i in enumerate((i0, i1, i2)))
    return ((a[:, None, None] * b[None, :, None]) * c[None, None, :]).astype(dt).astype(np.float64)


def moveout_axes(kind, ndim, nh, npp, nt, rng):
    """unitless axes whose curves cross the window, with known edges among them:
    - offsets irregular in [-8, 8] plus the dyadic 2, 4 and 4.75 (y: 0 and 4);
    - linear / parabolic p spanning +-1.5 nt over the window, plus dyadic p, so that some tdec are integers (d = 0)
      and tdec = nt - 1 exactly at (h, p) = (2, 1) / (2, 0.25) and t0 = nt - 3 / nt - 2;
    - hyperbolic p = 0, p = 1e-300 (q * q overflows), h / p up to 3 nt, and (4.75, 1/16): q = 76, so at nt = 96 the
      pair t0 = 57 lands on tdec = 95 = nt - 1 exactly;
    - in 3-D (linear / parabolic) a model pair whose terms at hx = hy = 4 are +1e17 and -1e17: cx + cy cancels to 0,
      while (t0 + cx) + cy rounds t0 to multiples of 16."""
    nhy, nhx = nh
    npy, npx = npp
    H = 8.0
    hx = np.sort(np.concatenate([rng.uniform(-H, H, nhx - 3), [2.0, 4.0, 4.75]]))
    if kind == "linear":
        px = np.concatenate([[1.0, -0.5, 0.0], rng.uniform(-1.5 * nt / H, 1.5 * nt / H, npx - 3)])
    elif kind == "parabolic":
        px = np.concatenate([[0.25, -0.0625, 0.0], rng.uniform(-1.5 * nt / H ** 2, 1.5 * nt / H ** 2, npx - 3)])
    else:
        px = np.concatenate([[0.0, 1e-300, 0.0625, 0.5], rng.uniform(H / (3 * nt), 2.0, npx - 4)])
    if ndim == 2:
        return None, hx, None, px
    hy = np.sort(np.concatenate([rng.uniform(-6, 6, nhy - 2), [0.0, 4.0]]))
    if kind == "hyperbolic":
        py = np.concatenate([[0.5, 1e-300], rng.uniform(6 / (3 * nt), 2.0, npy - 2)])
    else:
        big = 2.5e16 if kind == "linear" else 6.25e15
        scale = 1.5 * nt / (6.0 if kind == "linear" else 36.0)
        py = np.concatenate([[-1.0 if kind == "linear" else -0.25], rng.uniform(-scale, scale, npy - 2), [-big]])
        px = px.copy()
        px[-1] = big
    return hy, hx, py, px


# name: nt, (nhy, nhx), (npy, npx), then per window axis (y, x, t): (windows, step, traces or samples past the last)
GEOMS = {
    "moveout": (96, (4, 8), (3, 8), (2, 3, 1), (3, 5, 1), (3, 40, 5)),
    "overlap": (8, (8, 8), (3, 5), (4, 2, 1), (4, 2, 1), (4, 2, 1)),      # len 8, step 2: four windows per sample
    "edges": (16, (5, 6), (3, 4), (1, 1, 0), (2, 6, 1), (2, 16, 3)),      # nwin = n; step = len (no overlap)
    "wide": (5, (2, 300), (3, 270), (2, 1, 0), (2, 150, 1), (2, 3, 1)),   # 300 traces, 270 model traces
    "long": (600, (3, 6), (3, 5), (2, 2, 1), (2, 3, 1), (2, 300, 7)),     # 3 sample CTAs, len 600 % 256 != 0
}
ENTRY_GEOMS = {"radon": ["moveout", "wide", "long"], "windows": list(GEOMS), "patches": list(GEOMS)}


def make_geo(entry, geom, kind, interp, ndim, rng, tapered=True):
    nt, nh, npp, wy, wx, wt = GEOMS[geom]
    if ndim == 2:
        nh, npp, wy = (1, nh[1]), (1, npp[1]), (1, 1, 0)
    hy, hx, py, px = moveout_axes(kind, ndim, nh, npp, nt, rng)
    if entry == "radon":
        return Geo(entry, kind, interp, hy, hx, py, px, nt)
    if entry == "windows":
        wt = (1, 1, 0)
    Ls = (nh[0], nh[1], nt)
    ws = (wy, wx, wt)
    n = tuple((w[0] - 1) * w[1] + Ls[a] + w[2] for a, w in enumerate(ws))
    nw, st = tuple(w[0] for w in ws), tuple(w[1] for w in ws)
    taper = None
    if tapered and entry == "windows":
        taper = ("table", rng.uniform(0.05, 1.0, (nw[0] * nw[1], nh[0], nh[1])))
    elif tapered:
        taper = ("axis", [None if ndim == 2 else rng.uniform(0.05, 1.0, (nw[0], Ls[0])),
                          rng.uniform(0.05, 1.0, (nw[1], Ls[1])), rng.uniform(0.05, 1.0, (nw[2], Ls[2]))])
    return Geo(entry, kind, interp, hy, hx, py, px, nt, n, nw, st, taper)


# ---------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------
def tdec_all(kind, t0, hx, px, hy=None, py=None):
    """test_radon.tdec over broadcast arrays: the same IEEE operations in the same order, element by element"""
    t0 = np.asarray(t0, dtype=np.int64)
    with np.errstate(all="ignore"):
        if kind == "hyperbolic":
            q = hx / px
            v = (t0 * t0).astype(np.float64) + q * q
            if hy is not None:
                r = hy / py
                v = v + r * r
            return np.sqrt(v)
        cx = px * hx if kind == "linear" else px * (hx * hx)
        v = t0.astype(np.float64) + cx
        if hy is not None:
            v = v + (py * hy if kind == "linear" else py * (hy * hy))
        return v


def radon_sparse(kind, interp, nt, hx, px, hy=None, py=None):
    """test_radon.dense as float64 CSR: data (hy, hx, t) x model (py, px, t0)"""
    hx, px = np.asarray(hx, dtype=np.float64), np.asarray(px, dtype=np.float64)
    nhx, npx = len(hx), len(px)
    nhy, npy = (1, 1) if hy is None else (len(hy), len(py))
    shape = (nhy, nhx, npy, npx, nt)
    t0 = np.arange(nt).reshape(1, 1, 1, 1, nt)
    if hy is None:
        v = tdec_all(kind, t0, hx.reshape(1, nhx, 1, 1, 1), px.reshape(1, 1, 1, npx, 1))
    else:
        v = tdec_all(kind, t0, hx.reshape(1, nhx, 1, 1, 1), px.reshape(1, 1, 1, npx, 1),
                     np.asarray(hy, dtype=np.float64).reshape(nhy, 1, 1, 1, 1),
                     np.asarray(py, dtype=np.float64).reshape(1, 1, npy, 1, 1))
    v = np.broadcast_to(v, shape)
    ok = (v >= 0) & (v < (nt - 1 if interp else nt))
    jy, jx, iy, ix, tt = np.nonzero(ok)
    vv = v[ok]
    it = np.floor(vv).astype(np.int64)
    row = (jy * nhx + jx) * nt + it
    col = (iy * npx + ix) * nt + tt
    if interp:
        d = vv - it
        row, col, val = np.concatenate([row, row + 1]), np.concatenate([col, col]), np.concatenate([1 - d, d])
    else:
        val = np.ones(len(row))
    return sp.csr_matrix((val, (row, col)), shape=(nhy * nhx * nt, npy * npx * nt))


def geo_radon(G):
    return radon_sparse(G.kind, G.interp, G.L[2], G.hx, G.px, G.hy, G.py)


def window_matrix(G, A, dt):
    """sum_w R_w^T diag(tap_w) A_w as float64 CSR: section (n0, n1, ns) x window-major model; A is one window's
    operator, rows (jy, jx, sl), columns the window's model"""
    A = sp.coo_matrix(A)
    nhy, nhx, nt = G.L
    jy, r = np.divmod(A.row, nhx * nt)
    jx, sl = np.divmod(r, nt)
    rows, cols, vals = [], [], []
    for w, (i0, i1, i2) in enumerate(G.windows()):
        tap = np.ascontiguousarray(tap_window(G, dt, i0, i1, i2)).ravel()
        rows.append(((i0 * G.st[0] + jy) * G.n[1] + i1 * G.st[1] + jx) * G.n[2] + i2 * G.st[2] + sl)
        cols.append(w * A.shape[1] + A.col)
        vals.append(tap[A.row] * A.data)
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))),
                         shape=(G.nd, G.nwin * A.shape[1]))


def bound_coefficient(k, m, dt):
    return (k + 3) * U64 + (m + 2) * unit(dt) + k * ULD


def check_bound(got, ref, absref, k, m, dt, what):
    """|got - ref| <= bound_coefficient * absref componentwise; returns the worst ratio of error to bound"""
    c = bound_coefficient(k, m, dt)
    assert c < (1e-5 if dt == np.float32 else 1e-12), (what, k, m, c)
    tol = c * np.asarray(absref, dtype=np.float64)
    err = np.abs(np.asarray(got, dtype=np.float64) - np.asarray(ref, dtype=np.longdouble)).astype(np.float64)
    assert np.all(err <= tol), f"{what}: max err {err.max():.3e}, worst ratio {np.max(err / (tol + 1e-300)):.3f}"
    ratio = float(np.max(err / np.maximum(tol, 1e-300)))
    print(f"BOUND_RATIO {what} {ratio:.4f}")
    return ratio


def check_matrix(got, M, x, k, m, dt, what):
    """got (rows, C) against M x (float64 matrix, extended-precision product) under the bound"""
    ref = M.astype(np.longdouble) @ x.astype(np.longdouble)
    absref = abs(M) @ np.abs(x)
    return check_bound(got, ref, absref, k, m, dt, what)


def max_terms(A, adjoint):
    """the most terms in one window sum: nonzeros per row of A (forward) or per column (adjoint)"""
    A = sp.csr_matrix(A)
    return int(max(np.diff((A.T.tocsr() if adjoint else A).indptr).max(), 1))


def seq_sum(P):
    """the sums over axis 1 of P (rows, K, C), each accumulated term by term from 0.0 in float64"""
    acc = np.zeros((P.shape[0], P.shape[2]))
    for j in range(P.shape[1]):
        acc = acc + P[:, j]
    return acc


def forward_terms(G, jy, jx, Xw):
    """the float64 terms of window-local trace (jy, jx) at every window-local sample, in the order the forward adds
    them (model traces (py, px), t0 ascending): (nt, K, C), each row padded with zeros after its terms"""
    npy, npx = G.P
    nt = G.L[2]
    C = Xw.shape[-1]
    t0 = np.arange(nt).reshape(1, 1, nt)
    hy = None if G.hy is None else G.hy[jy]
    py = None if G.py is None else G.py.reshape(npy, 1, 1)
    v = np.broadcast_to(tdec_all(G.kind, t0, G.hx[jx], G.px.reshape(1, npx, 1), hy, py), (npy, npx, nt)).ravel()
    x = Xw.reshape(-1, C)
    idx = np.nonzero((v >= 0) & (v < (nt - 1 if G.interp else nt)))[0]
    vv = v[idx]
    it = np.floor(vv).astype(np.int64)
    if G.interp:
        d = vv - it
        samp, midx = np.concatenate([it, it + 1]), np.concatenate([idx, idx])
        val = np.concatenate([x[idx] * (1.0 - d)[:, None], x[idx] * d[:, None]])
    else:
        samp, midx, val = it, idx, x[idx]
    order = np.lexsort((midx, samp))
    samp, val = samp[order], val[order]
    counts = np.bincount(samp, minlength=nt)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    P = np.zeros((nt, max(int(counts.max(initial=0)), 1), C))
    P[samp, np.arange(len(samp)) - starts[samp]] = val
    return P


def emulate_forward(G, dt, X, traces):
    """the windowed forward at whole section traces ``traces`` [(a, b)], X the model [nw][npy][npx][nt][C] (values of
    T as float64).  Returns (out as T in float64, the extended-precision definition, sum of |terms| times |tap|,
    the most terms in one window sum), each [len(traces)][ns][C]"""
    ns, nt = G.n[2], G.L[2]
    C = X.shape[-1]
    X = X.reshape(G.nwin, -1, C)
    out = np.zeros((len(traces), ns, C))
    ref = np.zeros((len(traces), ns, C), dtype=np.longdouble)
    bnd = np.zeros((len(traces), ns, C))
    kmax = 1
    for n_, (a, b) in enumerate(traces):
        o = np.zeros((ns, C), dtype=dt)
        for i0 in G.covering(0, a):
            part = np.zeros((ns, C), dtype=dt)
            for i1 in G.covering(1, b):
                jy, jx = a - i0 * G.st[0], b - i1 * G.st[1]
                q = np.zeros((ns, C), dtype=dt)
                for i2 in range(G.nw[2]):
                    w = (i0 * G.nw[1] + i1) * G.nw[2] + i2
                    P = forward_terms(G, jy, jx, X[w])
                    kmax = max(kmax, int(np.count_nonzero(np.abs(P).sum(2), 1).max()))
                    tap = tap_window(G, dt, i0, i1, i2)[jy, jx]
                    s = slice(i2 * G.st[2], i2 * G.st[2] + nt)
                    q[s] = q[s] + tap.astype(dt)[:, None] * seq_sum(P).astype(dt)
                    ref[n_, s] += tap[:, None] * P.astype(np.longdouble).sum(1)
                    bnd[n_, s] += tap[:, None] * np.abs(P).sum(1)
                part = part + q
            o = o + part
        out[n_] = o
    return out, ref, bnd, kmax


def emulate_adjoint(G, dt, D, mtraces):
    """the windowed adjoint at whole model traces ``mtraces`` [(w, ipy, ipx)], D the section [n0][n1][ns][C]
    (values of T as float64).  Returns (out, definition, sum of |terms|, most terms), each [len(mtraces)][nt][C]"""
    nhy, nhx, nt = G.L
    C = D.shape[-1]
    D = D.reshape(*G.n, C)
    lim = nt - 1 if G.interp else nt
    out = np.zeros((len(mtraces), nt, C))
    ref = np.zeros((len(mtraces), nt, C), dtype=np.longdouble)
    bnd = np.zeros((len(mtraces), nt, C))
    kmax = 1
    t0 = np.arange(nt)
    for w in sorted({m[0] for m in mtraces}):
        sel = [j for j, m in enumerate(mtraces) if m[0] == w]
        ipy = np.array([mtraces[j][1] for j in sel])[:, None]
        ipx = np.array([mtraces[j][2] for j in sel])[:, None]
        i0, i1, i2 = np.unravel_index(w, G.nw)
        a0, b0, o2 = i0 * G.st[0], i1 * G.st[1], i2 * G.st[2]
        tapw = tap_window(G, dt, i0, i1, i2)
        acc = np.zeros((len(sel), nt, C))
        racc = np.zeros((len(sel), nt, C), dtype=np.longdouble)
        bacc = np.zeros((len(sel), nt, C))
        cnt = np.zeros((len(sel), nt), dtype=np.int64)
        for jy in range(nhy):
            hy = None if G.hy is None else G.hy[jy]
            py = None if G.py is None else G.py[ipy]
            for jx in range(nhx):
                v = tdec_all(G.kind, t0[None, :], G.hx[jx], G.px[ipx], hy, py)
                v = np.broadcast_to(v, (len(sel), nt))
                ok = (v >= 0) & (v < lim)
                if not ok.any():
                    continue
                r, c = np.nonzero(ok)
                vv = v[ok]
                it = np.floor(vv).astype(np.int64)
                trace = D[a0 + jy, b0 + jx, o2:o2 + nt]
                tp = tapw[jy, jx]
                x0 = (tp[it].astype(dt)[:, None] * trace[it].astype(dt)).astype(np.float64)
                e0 = tp[it, None].astype(np.longdouble) * trace[it]
                if G.interp:
                    d = vv - it
                    w0 = 1.0 - d
                    x1 = (tp[it + 1].astype(dt)[:, None] * trace[it + 1].astype(dt)).astype(np.float64)
                    e1 = tp[it + 1, None].astype(np.longdouble) * trace[it + 1]
                    term = x0 * w0[:, None] + x1 * d[:, None]
                    racc[r, c] += e0 * w0[:, None] + e1 * d[:, None]
                    bacc[r, c] += np.abs(e0).astype(np.float64) * w0[:, None] + np.abs(e1).astype(np.float64) * d[:, None]
                    cnt[r, c] += 2
                else:
                    term = x0
                    racc[r, c] += e0
                    bacc[r, c] += np.abs(e0).astype(np.float64)
                    cnt[r, c] += 1
                acc[r, c] = acc[r, c] + term
        out[sel] = acc.astype(dt)
        ref[sel], bnd[sel] = racc, bacc
        kmax = max(kmax, int(cnt.max()))
    return out, ref, bnd, kmax


def sample_traces(G, C, rng, need=512):
    """whole section traces to emulate: the first, the last (past the last window where the geometry has such
    traces), one held by the most windows, then random ones until ``need`` outputs"""
    n0, n1, ns = G.n
    deep = tuple(max(range(G.n[ax]), key=lambda a: len(G.covering(ax, a))) for ax in (0, 1))
    tr = [(0, 0), (n0 - 1, n1 - 1), deep]
    past = [(a, b) for a, b in itertools.product(range(n0), range(n1)) if not G.covering(0, a) or not G.covering(1, b)]
    tr += past[:1]
    rest = list(itertools.product(range(n0), range(n1)))
    for j in rng.permutation(len(rest)):
        if len(set(tr)) * ns * C >= need:
            break
        tr.append(rest[j])
    return list(dict.fromkeys(tr))


def sample_mtraces(G, C, rng, need=512):
    """whole model traces to emulate: the first and last of the model, then random ones of a few windows"""
    npy, npx = G.P
    mt = [(0, 0, 0), (G.nwin - 1, npy - 1, npx - 1)]
    rest = list(itertools.product(sorted({0, G.nwin - 1, int(rng.integers(G.nwin))}), range(npy), range(npx)))
    rest += list(itertools.product(range(G.nwin), range(npy), range(npx)))
    for j in np.concatenate([rng.permutation(len(rest) - G.nwin * npy * npx),
                             len(rest) - G.nwin * npy * npx + rng.permutation(G.nwin * npy * npx)]):
        if len(set(mt)) * G.L[2] * C >= need:
            break
        mt.append(rest[j])
    return list(dict.fromkeys(mt))


# ---------------------------------------------------------------------------------------------------------------
# CPU: the references against each other
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.filterwarnings("ignore:overflow encountered")
@pytest.mark.parametrize("interp", [True, False], ids=["interp", "nointerp"])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("ndim", [2, 3], ids=["2d", "3d"])
def test_radon_sparse_is_the_dense_definition(ndim, kind, interp):
    """at test_radon's KERNEL_SHAPES and at the large-moveout axes (p = 0, p = 1e-300, a cancelling 3-D pair)"""
    rng = np.random.default_rng(100 + 10 * ndim + 2 * KINDS.index(kind) + int(interp))
    cases = [(nt, kernel_axes(kind, ndim, rng, nhs, nps)) for nt, nhs, nps in KERNEL_SHAPES]
    cases.append((96, moveout_axes(kind, ndim, (3, 8), (3, 6), 96, rng)))
    for nt, (hy, hx, py, px) in cases:
        M = dense(kind, interp, nt, hx, px, hy, py)
        S = radon_sparse(kind, interp, nt, hx, px, hy, py)
        assert S.shape == M.shape
        np.testing.assert_array_equal(S.toarray(), M, err_msg=f"nt={nt} {len(hx)}x{len(px)}")
    assert np.count_nonzero(M) > 0


def test_moveout_axes_reach_their_edges():
    """the large-moveout axes hold what the probes rely on: integer tdec, tdec = nt - 1, pairs past both ends of the
    window, p whose terms overflow, and (3-D) the cancelling pair"""
    rng = np.random.default_rng(5)
    for kind in KINDS:
        for ndim in (2, 3):
            hy, hx, py, px = moveout_axes(kind, ndim, (4, 8), (3, 8), 96, rng)
            G = Geo("radon", kind, True, hy, hx, py, px, 96)
            t0 = np.arange(96).reshape(1, 1, 1, 1, 96)
            v = tdec_all(kind, t0, hx.reshape(1, -1, 1, 1, 1), px.reshape(1, 1, 1, -1, 1),
                         None if hy is None else hy.reshape(-1, 1, 1, 1, 1),
                         None if py is None else py.reshape(1, 1, -1, 1, 1))
            v = np.broadcast_to(v, (G.L[0], G.L[1], G.P[0], G.P[1], 96))
            fin = v[np.isfinite(v)]
            assert np.any(v == 95.0), (kind, ndim)
            assert np.any((fin == np.floor(fin)) & (fin < 95)), (kind, ndim)
            assert np.any(fin >= 96) and (kind == "hyperbolic" or np.any(fin < 0))
            if kind == "hyperbolic":
                assert np.any(~np.isfinite(v))
            if ndim == 3 and kind != "hyperbolic":
                assert np.any(np.isin(v[:, :, -1, -1][np.isin(hy, [4.0])][:, np.isin(hx, [4.0])], [16.0, 32.0]))


@pytest.mark.parametrize("shape", test_patch.PATCH_SHAPES, ids=[str(s[0]) for s in test_patch.PATCH_SHAPES])
def test_window_matrix_is_the_fold_of_window_products_patch(shape):
    """window_matrix against test_patch.fold_ref of the per-window products, per-axis tapers, within the float64
    bound"""
    n, nw, L, st, ni = shape
    rng = np.random.default_rng(sum(n))
    taps = [rng.uniform(0, 1, (nw[a], L[a])) if (a == 2 or n[a] > 1) else None for a in range(3)]
    A = sp.random(int(np.prod(L)), 3, density=0.6, random_state=int(sum(L)), format="csr")
    G = Geo("patches", "linear", False, None, np.zeros(L[1]), None, np.zeros(3), L[2], n, nw, st, ("axis", taps))
    G.L = tuple(L)
    X = rng.standard_normal((int(np.prod(nw)), 3, ni))
    win = np.stack([A @ X[w] for w in range(len(X))])
    ref = test_patch.fold_ref(win.ravel(), n, nw, L, st, ni, taps, np.float64).reshape(-1, ni)
    W = window_matrix(G, A, np.float64)
    check_matrix(ref, W, X.reshape(-1, ni), max_terms(A, False), G.depth(), np.float64, "fold_ref-patch")


@pytest.mark.parametrize("shape", test_sliding.SLIDING_SHAPES[:4] + test_sliding.SLIDING_SHAPES[5:],
                         ids=lambda s: str(s[0]))
def test_window_matrix_is_the_fold_of_window_products_sliding(shape):
    """window_matrix against test_sliding.fold_ref of the per-window products, T-table tapers, within the float64
    bound"""
    n, nw, L, st, nt, ni = shape
    rng = np.random.default_rng(sum(n) + nt)
    tab = rng.uniform(0, 1, (nw[0] * nw[1], L[0], L[1]))
    A = sp.random(L[0] * L[1] * nt, 4, density=0.6, random_state=nt, format="csr")
    G = Geo("windows", "linear", False, None, np.zeros(L[1]), None, np.zeros(4), nt, (n[0], n[1], nt),
            (nw[0], nw[1], 1), (st[0], st[1], 1), ("table", tab))
    G.L = (L[0], L[1], nt)
    X = rng.standard_normal((nw[0] * nw[1], 4, ni))
    win = np.stack([A @ X[w] for w in range(len(X))])
    ref = test_sliding.fold_ref(win.ravel(), n[0], n[1], nt * ni, nw, L, st, tab, np.float64).reshape(-1, ni)
    W = window_matrix(G, A, np.float64)
    check_matrix(ref, W, X.reshape(-1, ni), max_terms(A, False), G.depth(), np.float64, "fold_ref-sliding")


SELF_CASES = [(e, g) for e in ("radon", "windows", "patches") for g in ("moveout", "overlap", "edges")
              if g in ENTRY_GEOMS[e]]


@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("case", SELF_CASES, ids=[f"{e}-{g}" for e, g in SELF_CASES])
def test_emulation_is_the_window_matrix(case, dt):
    """emulate_forward / emulate_adjoint against window_matrix within the bound, for every kind, interp and 2-D /
    3-D: the emulation's order of operations is a valid evaluation of the definition"""
    entry, geom = case
    rng = np.random.default_rng(7 + ["radon", "windows", "patches"].index(entry))
    for kind, interp, ndim in itertools.product(KINDS, (True, False), (2, 3)):
        G = make_geo(entry, geom, kind, interp, ndim, rng)
        A = geo_radon(G)
        W = window_matrix(G, A, dt)
        C = 2 if dt == np.float64 else 1
        X = rng.standard_normal((G.nwin * G.nm, C)).astype(dt).astype(np.float64)
        tr = sample_traces(G, C, rng, need=64)
        got, _, _, k = emulate_forward(G, dt, X, tr)
        assert k <= max_terms(A, False)
        rows = np.concatenate([(a * G.n[1] + b) * G.n[2] + np.arange(G.n[2]) for a, b in tr])
        check_matrix(got.reshape(-1, C), W[rows], X, max_terms(A, False), G.depth(), dt, "emulation-fwd")
        D = rng.standard_normal((G.nd, C)).astype(dt).astype(np.float64)
        mt = sample_mtraces(G, C, rng, need=64)
        got, _, _, k = emulate_adjoint(G, dt, D, mt)
        assert k <= max_terms(A, True)
        rows = np.concatenate([w * G.nm + (iy * G.P[1] + ix) * G.L[2] + np.arange(G.L[2]) for w, iy, ix in mt])
        check_matrix(got.reshape(-1, C), W.T.tocsr()[rows], D, max_terms(A, True), 0, dt, "emulation-adj")


# ---------------------------------------------------------------------------------------------------------------
# GPU: the entry points through the C ABI
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


def dev(a, dt=np.float64):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a, dtype=dt)).cuda()


class Device:
    """G's axes and tapers on the device for data type dt (kept alive with the object)"""

    def __init__(self, G, dt):
        self.ax = [None if a is None else dev(a) for a in (G.hy, G.hx, G.py, G.px)]
        self.axp = [None if a is None else a.data_ptr() for a in self.ax]
        self.tap, self.tapp = [], [None, None, None]
        if G.taper is not None and G.taper[0] == "table":
            self.tap = [dev(G.taper[1], dt)]
            self.tapp = [self.tap[0].data_ptr()]
        elif G.taper is not None:
            self.tap = [None if t is None else dev(t) for t in G.taper[1]]
            self.tapp = [None if t is None else t.data_ptr() for t in self.tap]
        elif G.entry == "windows":
            self.tapp = [None]


def launch(pm, G, D, x, y, C, adjoint, dt):
    L = pm._lib
    code = L.F32 if dt == np.float32 else L.F64
    nhy, nhx, nt = G.L
    npy, npx = G.P
    k = KINDS.index(G.kind)
    if G.entry == "radon":
        return L.lib.b2_radon(L.ctx(), x, y, nt, C, nhy, nhx, npy, npx, *D.axp, k, int(G.interp), int(adjoint), code,
                              L.stream())
    if G.entry == "windows":
        return L.lib.b2_radon_windows(L.ctx(), x, y, nt, C, G.n[0], G.n[1], nhy, nhx, npy, npx, *D.axp, k,
                                      int(G.interp), G.nw[0], G.nw[1], G.st[0], G.st[1], D.tapp[0], int(adjoint), code,
                                      L.stream())
    return L.lib.b2_radon_patches(L.ctx(), x, y, nt, C, G.n[0], G.n[1], G.n[2], nhy, nhx, npy, npx, *D.axp, k,
                                  int(G.interp), *G.nw, *G.st, *D.tapp, int(adjoint), code, L.stream())


def run(pm, G, D, x, C, adjoint, dt):
    """one launch into a guarded, misaligned output, twice; x the input's values of T (float64, any shape).
    Returns the output as float64, (rows, C)"""
    xd = dev(np.asarray(x).ravel(), dt)
    n = (G.nwin * G.nm if adjoint else G.nd) * C
    got, guards, same = guarded_twice(lambda yp: launch(pm, G, D, xd.data_ptr(), yp, C, adjoint, dt), n, dt, 3,
                                      offset=1)
    assert guards and same
    return got.astype(np.float64).reshape(-1, C)


def route(pm, G, D, x, C, adjoint, dt):
    """b2_radon per window plus b2_sliding / b2_patch: the per-window route the fused entry points equal"""
    import torch
    L = pm._lib
    code = L.F32 if dt == np.float32 else L.F64
    nhy, nhx, nt = G.L
    npy, npx = G.P
    nwd, nm = nhy * nhx * nt * C, G.nm * C
    xd = dev(np.asarray(x).ravel(), dt)
    work = torch.empty(G.nwin * nwd, dtype=xd.dtype, device="cuda")
    out = torch.empty(G.nwin * nm if adjoint else G.nd * C, dtype=xd.dtype, device="cuda")

    def fold(src, dst, adj):
        if G.entry == "windows":
            rc = L.lib.b2_sliding(L.ctx(), src.data_ptr(), dst.data_ptr(), G.n[0], G.n[1], nt, C, G.nw[0], G.nw[1],
                                  nhy, nhx, G.st[0], G.st[1], D.tapp[0], adj, code, L.stream())
        else:
            rc = L.lib.b2_patch(L.ctx(), src.data_ptr(), dst.data_ptr(), *G.n, C, *G.nw, *G.L, *G.st, *D.tapp, adj,
                                code, L.stream())
        assert rc == 0

    if adjoint:
        fold(xd, work, 1)
    for w in range(G.nwin):
        src, dst = (work[w * nwd:], out[w * nm:]) if adjoint else (xd[w * nm:], work[w * nwd:])
        assert L.lib.b2_radon(L.ctx(), src.data_ptr(), dst.data_ptr(), nt, C, nhy, nhx, npy, npx, *D.axp,
                              KINDS.index(G.kind), int(G.interp), int(adjoint), code, L.stream()) == 0
    if not adjoint:
        fold(work, out, 0)
    return host(out).astype(np.float64).reshape(-1, C)


# ---- spike probes -----------------------------------------------------------------------------------------------
def forward_probes(G, rng):
    """model samples (w, ipy, ipx, t0): the first and last of the model, t0 = 0 and nt - 1, a window held by the most
    windows, p = 0 and p = 1e-300 (hyperbolic: px[0], px[1]), a pair that lands on tdec = nt - 1 or on an integer
    tdec, random ones"""
    npy, npx = G.P
    nt = G.L[2]
    mid = int(np.ravel_multi_index(tuple(v // 2 for v in G.nw), G.nw))
    pr = [(0, 0, 0, 0), (G.nwin - 1, npy - 1, npx - 1, nt - 1), (mid, 0, 1, nt // 2), (0, npy - 1, 0, nt // 3)]
    t0 = np.arange(nt).reshape(1, 1, 1, 1, nt)
    hy = None if G.hy is None else G.hy.reshape(-1, 1, 1, 1, 1)
    py = None if G.py is None else G.py.reshape(1, 1, -1, 1, 1)
    v = np.broadcast_to(tdec_all(G.kind, t0, G.hx.reshape(1, -1, 1, 1, 1), G.px.reshape(1, 1, 1, -1, 1), hy, py),
                        (*G.L[:2], *G.P, nt))
    for target in (v == nt - 1, (v == np.floor(v)) & (v < nt - 1) & (v > 0)):
        hit = np.argwhere(target)
        if len(hit):
            _, _, iy, ix, t = hit[len(hit) // 2]
            pr.append((mid, int(iy), int(ix), int(t)))
    for _ in range(2):
        pr.append((int(rng.integers(G.nwin)), int(rng.integers(npy)), int(rng.integers(npx)), int(rng.integers(nt))))
    return pr


def adjoint_probes(G, rng):
    """section samples (a, b, s): the first sample of the first window, the last of the last window, a sample held
    by the most windows, traces and samples past the last window, the last sample of a window, random ones"""
    n0, n1, ns = G.n
    deep = tuple(max(range(G.n[ax]), key=lambda a: len(G.covering(ax, a))) for ax in range(3))
    last = tuple((G.nw[ax] - 1) * G.st[ax] + G.L[ax] - 1 for ax in range(3))
    pr = [(0, 0, 0), last, deep, (0, deep[1], G.L[2] - 1), (n0 - 1, n1 - 1, deep[2]), (deep[0], deep[1], ns - 1)]
    for _ in range(2):
        pr.append((int(rng.integers(n0)), int(rng.integers(n1)), int(rng.integers(ns))))
    return pr


def predict_forward(G, Acsc, dt, C, probe, c, val):
    """the forward of a spike of val at model sample probe, component c: one term per output sample,
    mul_rn(tap, (T)(w * val))"""
    w, ipy, ipx, t0 = probe
    out = np.zeros((*G.n, C), dtype=dt)
    i0, i1, i2 = np.unravel_index(w, G.nw)
    col = (ipy * G.P[1] + ipx) * G.L[2] + t0
    rows = Acsc.indices[Acsc.indptr[col]:Acsc.indptr[col + 1]]
    wts = Acsc.data[Acsc.indptr[col]:Acsc.indptr[col + 1]]
    jy, r = np.divmod(rows, G.L[1] * G.L[2])
    jx, sl = np.divmod(r, G.L[2])
    tap = tap_window(G, dt, i0, i1, i2)[jy, jx, sl].astype(dt)
    out[i0 * G.st[0] + jy, i1 * G.st[1] + jx, i2 * G.st[2] + sl, c] = tap * (wts * val).astype(dt)
    return out.reshape(-1, C).astype(np.float64)


def predict_adjoint(G, Acsr, dt, C, probe, c, val):
    """the adjoint of a spike of val at section sample probe, component c: one term per model sample,
    (T)(w * (T)(tap * val))"""
    a, b, s = probe
    out = np.zeros((G.nwin, G.nm, C), dtype=dt)
    for i0, i1, i2 in itertools.product(G.covering(0, a), G.covering(1, b), G.covering(2, s)):
        jy, jx, sl = a - i0 * G.st[0], b - i1 * G.st[1], s - i2 * G.st[2]
        row = (jy * G.L[1] + jx) * G.L[2] + sl
        cols = Acsr.indices[Acsr.indptr[row]:Acsr.indptr[row + 1]]
        wts = Acsr.data[Acsr.indptr[row]:Acsr.indptr[row + 1]]
        xv = dt(tap_window(G, dt, i0, i1, i2)[jy, jx, sl]) * dt(val)
        out[int(np.ravel_multi_index((i0, i1, i2), G.nw)), cols, c] = (wts * np.float64(xv)).astype(dt)
    return out.reshape(-1, C).astype(np.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("entry", ["radon", "windows", "patches"])
def test_spike_probes_bitwise(pm, entry, kind):
    """a spike gives exactly one term per output sample, so the whole output is known bit for bit: index, weight,
    taper and window-covering errors show without any rounding tolerance"""
    rng = np.random.default_rng(300 + 10 * KINDS.index(kind) + ["radon", "windows", "patches"].index(entry))
    count = 0
    for geom in (["moveout", "long"] if entry == "radon" else ["moveout", "overlap"]):
        for ndim, interp in itertools.product((2, 3), (True, False)):
            G = make_geo(entry, geom, kind, interp, ndim, rng)
            A = geo_radon(G)
            Acsc, Acsr = A.tocsc(), A.tocsr()
            for dt, C in itertools.product((np.float32, np.float64), (1, 2)):
                D = Device(G, dt)
                val = np.float64(dt(SPIKE))
                for adjoint in (False, True):
                    probes = adjoint_probes(G, rng) if adjoint else forward_probes(G, rng)
                    for probe in probes:
                        c = C - 1
                        x = np.zeros(((G.nd if adjoint else G.nwin * G.nm), C))
                        if adjoint:
                            x.reshape(*G.n, C)[probe + (c,)] = val
                            want = predict_adjoint(G, Acsr, dt, C, probe, c, val)
                        else:
                            w, iy, ix, t = probe
                            x.reshape(G.nwin, *G.P, G.L[2], C)[w, iy, ix, t, c] = val
                            want = predict_forward(G, Acsc, dt, C, probe, c, val)
                        got = run(pm, G, D, x, C, adjoint, dt)
                        np.testing.assert_array_equal(
                            got, want, err_msg=f"{geom} {ndim}d interp={interp} {np.dtype(dt).name} C={C} "
                                               f"adj={adjoint} probe={probe}")
                        count += 1
    assert count >= 300


# ---- random inputs ------------------------------------------------------------------------------------------------
CASES = [(e, g) for e in ("radon", "windows", "patches") for g in ENTRY_GEOMS[e]]
DT_CASES = [(np.float32, 1, True), (np.float64, 2, True), (np.float64, 1, False)]   # (T, n_inner, tapered)
# the wide windows (300 traces, 270 model traces) skip the third, untapered case: the time goes to the others


@pytest.mark.gpu
@pytest.mark.parametrize("ndim", [2, 3], ids=["2d", "3d"])
@pytest.mark.parametrize("interp", [True, False], ids=["interp", "nointerp"])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", CASES, ids=[f"{e}-{g}" for e, g in CASES])
def test_random_inputs_bound_emulation_and_route(pm, case, kind, interp, ndim):
    """random inputs: every output against window_matrix under the bound, at least 512 outputs (whole first, last
    and uncovered traces) against the emulation bit for bit, and the fused entry points against the per-window
    route bit for bit"""
    entry, geom = case
    seed = 1000 + 100 * CASES.index(case) + 10 * KINDS.index(kind) + 2 * int(interp) + ndim
    rng = np.random.default_rng(seed)
    for dt, C, tapered in (DT_CASES[:2] if geom == "wide" else DT_CASES):
        G = make_geo(entry, geom, kind, interp, ndim, rng, tapered)
        D = Device(G, dt)
        A = geo_radon(G)
        full = A.nnz * G.nwin <= 4_000_000       # the whole window_matrix; past that size, the sampled outputs
        W = window_matrix(G, A, dt) if full else None
        what = f"{entry} {geom} {kind} interp={interp} {ndim}d {np.dtype(dt).name} C={C} tapered={tapered}"
        for adjoint in (False, True):
            x = rng.standard_normal(((G.nd if adjoint else G.nwin * G.nm), C)).astype(dt).astype(np.float64)
            got = run(pm, G, D, x, C, adjoint, dt)
            tag = f"{entry} {'adj' if adjoint else 'fwd'} {np.dtype(dt).name}"
            m = 0 if adjoint else G.depth()
            if full:
                check_matrix(got, W.T.tocsr() if adjoint else W, x, max_terms(A, adjoint), m, dt, tag)
            if adjoint:
                mt = sample_mtraces(G, C, rng)
                emu, ref, bnd, k = emulate_adjoint(G, dt, x, mt)
                rows = np.concatenate([(w * G.nm + (iy * G.P[1] + ix) * G.L[2]) + np.arange(G.L[2])
                                       for w, iy, ix in mt])
            else:
                tr = sample_traces(G, C, rng)
                emu, ref, bnd, k = emulate_forward(G, dt, x, tr)
                rows = np.concatenate([(a * G.n[1] + b) * G.n[2] + np.arange(G.n[2]) for a, b in tr])
            assert emu.size >= 512 or emu.size == got.size
            if not full:
                check_bound(got[rows], ref.reshape(-1, C), bnd.reshape(-1, C), k, m, dt, tag)
            np.testing.assert_array_equal(got[rows], emu.reshape(-1, C), err_msg=f"{what} adj={adjoint} emulation")
            if entry != "radon":
                np.testing.assert_array_equal(got, route(pm, G, D, x, C, adjoint, dt),
                                              err_msg=f"{what} adj={adjoint} route")


# ---- b2_patch past the block limit ----------------------------------------------------------------------------------
def fold_levels(win, n, nw, L, st, taps, dt):
    """b2_patch's forward, vectorised over window samples: each (i0, i1)'s windows summed over i2 into a partial
    block, those summed over i1, then over i0, every product and sum in dt and in that order (a sample outside a
    window adds nothing: its partial sums stay where they were)"""
    ni = win.shape[-1]
    win = win.reshape(*nw, *L, ni)
    out = np.zeros((*n, ni), dtype=dt)
    for i0 in range(nw[0]):
        part = np.zeros((L[0], n[1], n[2], ni), dtype=dt)
        for i1 in range(nw[1]):
            q = np.zeros((L[0], L[1], n[2], ni), dtype=dt)
            t01 = taps[0][i0][:, None] * taps[1][i1][None, :]
            for i2 in range(nw[2]):
                tap = (t01[:, :, None] * taps[2][i2][None, None, :]).astype(dt)
                s = slice(i2 * st[2], i2 * st[2] + L[2])
                q[:, :, s] = q[:, :, s] + tap[..., None] * win[i0, i1, i2]
            s = slice(i1 * st[1], i1 * st[1] + L[1])
            part[:, s] = part[:, s] + q
        s = slice(i0 * st[0], i0 * st[0] + L[0])
        out[s] = out[s] + part
    return out


def unfold_levels(d, n, nw, L, st, taps, dt):
    ni = d.shape[-1]
    d = d.reshape(*n, ni)
    out = np.empty((*nw, *L, ni), dtype=dt)
    for i0, i1 in itertools.product(range(nw[0]), range(nw[1])):
        t01 = taps[0][i0][:, None] * taps[1][i1][None, :]
        blk = d[i0 * st[0]:i0 * st[0] + L[0], i1 * st[1]:i1 * st[1] + L[1]]
        for i2 in range(nw[2]):
            tap = (t01[:, :, None] * taps[2][i2][None, None, :]).astype(dt)
            out[i0, i1, i2] = tap[..., None] * blk[:, :, i2 * st[2]:i2 * st[2] + L[2]]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
def test_patch_kernel_past_the_block_limit(pm, dt):
    """b2_patch with more than 2^16 CTAs of 256 values in both directions (the grid-stride loop runs several
    rounds), time windows three deep, overlapping trace windows, a sample past the last window, all three axes
    tapered; bit for bit against the vectorised level-by-level fold"""
    n, nw, L, st, ni = (3, 18, 320_001), (2, 3, 3198), (2, 6, 300), (1, 6, 100), 1
    rng = np.random.default_rng(21)
    assert np.prod(n) * ni > (1 << 16) * 256
    taps = [rng.uniform(0.05, 1.0, (nw[a], L[a])) for a in range(3)]
    td = [dev(t) for t in taps]
    code = pm._lib.F32 if dt == np.float32 else pm._lib.F64
    nwv, ndv = int(np.prod(nw) * np.prod(L)) * ni, int(np.prod(n)) * ni
    for adjoint in (False, True):
        x = rng.standard_normal((ndv if adjoint else nwv, ni)).astype(dt)
        xd = dev(x, dt)
        got, guards, same = guarded_twice(
            lambda yp: test_patch.c_patch(pm, xd.data_ptr(), yp, *n, ni, *nw, *L, *st, *[t.data_ptr() for t in td],
                                          int(adjoint), code), nwv if adjoint else ndv, dt, 3, offset=1)
        assert guards and same
        want = (unfold_levels if adjoint else fold_levels)(x, n, nw, L, st, taps, dt)
        np.testing.assert_array_equal(got, want.ravel(), err_msg=f"adjoint={adjoint}")
        del x, xd, got, want


# ---- the benchmark's patch operators --------------------------------------------------------------------------------
PDT, PDH = 0.004, 12.5                                   # bench_patch.py's sampling and its p ranges
P_RANGE = {"linear": (-1.2e-3, 1.2e-3), "hyperbolic": (1500.0, 4500.0)}
PRODUCTION = ["2d-linear-float32", "2d-linear-float64", "2d-hyperbolic-float32", "2d-hyperbolic-float64",
              "3d-linear-float32"]


def production(pm, case):
    """(the Patch operator, its Radon, the physical (h, p) axes) of bench_patch.py's geometries"""
    L = pm.local
    ndim, kind, dt = case.split("-")
    if ndim == "2d":
        nwin, nover, npp = (64, 128), (32, 64), 64
        h, p = np.arange(nwin[0]) * PDH, np.linspace(*P_RANGE[kind], npp)
        R = L.Radon2D(np.arange(nwin[1]) * PDT, h, p, kind=kind, dtype=dt)
        _, dims, _, _ = L.patch2d_design((1024, 1024), nwin, nover, (npp, nwin[1]))
        return L.Patch2D(R, dims, (1024, 1024), nwin, nover, (npp, nwin[1])), R, [(h, p)]
    nwin, nover, npp = (32, 32, 64), (16, 16, 32), (16, 16)
    hs = [np.arange(nwin[a]) * PDH for a in (0, 1)]
    ps = [np.linspace(-1e-3, 1e-3, npp[a]) for a in (0, 1)]
    R = L.Radon3D(np.arange(nwin[2]) * PDT, *hs, *ps, dtype=dt)
    _, dims, _, _ = L.patch3d_design((128, 128, 256), nwin, nover, (*npp, nwin[2]))
    return L.Patch3D(R, dims, (128, 128, 256), nwin, nover, (*npp, nwin[2])), R, list(zip(hs, ps))


@pytest.mark.gpu
@pytest.mark.parametrize("case", PRODUCTION)
def test_production_patch_operators(pm, case):
    """Patch2D / Patch3D over Radon2D / Radon3D at bench_patch.py's geometries through the public API: the unitless
    axes, sampled outputs against the emulation (bit for bit) and the float64 definition (bound), and the fused apply
    against the per-patch route, bit for bit, real and complex128"""
    import torch
    S, R, phys = production(pm, case)
    assert S._fused is R
    kind, dt = R.kind, np.dtype(R.dtype).type
    axes = [unitless(kind, PDT, h, p, True) for h, p in phys]
    want = [a[0] for a in axes] + [a[1] for a in axes]
    got_axes = [host(a) for a in R._axes]
    for g, w in zip(got_axes, want):
        np.testing.assert_array_equal(g, w)
    if len(phys) == 1:
        hy, hx, py, px = None, got_axes[0], None, got_axes[1]
    else:
        hy, hx, py, px = got_axes
    taps = [None if t is None else host(t) for t in S._taps]
    G = Geo("patches", kind, R.interp, hy, hx, py, px, R._nt, S._section, S._nwins, S._steps, ("axis", taps))
    assert G.L == tuple(S._nwin)
    rng = np.random.default_rng(PRODUCTION.index(case))
    tdt = torch.float32 if dt == np.float32 else torch.float64
    for adjoint in (False, True):
        x = rng.standard_normal(S.shape[0] if adjoint else S.shape[1]).astype(dt)
        xt = torch.as_tensor(x).cuda()
        got = host(S.rmatvec(xt) if adjoint else S.matvec(xt)).astype(np.float64)
        x64 = x.astype(np.float64)[:, None]
        if adjoint:
            mt = [(0, 0, 0), (G.nwin - 1, G.P[0] - 1, G.P[1] - 1)]
            mt += [(w, int(rng.integers(G.P[0])), int(rng.integers(G.P[1])))
                   for w in (0, G.nwin // 2, G.nwin - 1) for _ in range(3)]
            emu, ref, bnd, k = emulate_adjoint(G, dt, x64, mt)
            rows = np.concatenate([w * G.nm + (iy * G.P[1] + ix) * G.L[2] + np.arange(G.L[2]) for w, iy, ix in mt])
        else:
            tr = [(0, 0), (G.n[0] - 1, G.n[1] - 1), (G.n[0] // 2, G.n[1] // 2 + 1)]
            emu, ref, bnd, k = emulate_forward(G, dt, x64, tr)
            rows = np.concatenate([(a * G.n[1] + b) * G.n[2] + np.arange(G.n[2]) for a, b in tr])
        assert emu.size >= 512
        np.testing.assert_array_equal(got[rows], emu.ravel(), err_msg=f"{case} adjoint={adjoint} emulation")
        check_bound(got[rows], ref.ravel(), bnd.ravel(), k, 0 if adjoint else G.depth(), dt,
                    f"production-{case} {'adj' if adjoint else 'fwd'}")
        U = copy.copy(S)
        U._fused, U._work = None, {}
        for data in (xt, torch.complex(xt.double(), torch.as_tensor(rng.standard_normal(x.size)).cuda())):
            a = S.rmatvec(data) if adjoint else S.matvec(data)
            b = U.rmatvec(data) if adjoint else U.matvec(data)
            assert a.dtype == b.dtype and (data.is_complex() or a.dtype == tdt)
            assert torch.equal(a, b), f"{case} adjoint={adjoint} {data.dtype}: fused != per-patch route"


# ---------------------------------------------------------------------------------------------------------------
# GPU: the operators with three or more windows over a sample
# ---------------------------------------------------------------------------------------------------------------
OPERATORS = [(c, i) for c in ("Sliding2D", "Sliding3D", "Patch2D", "Patch3D") for i in ("radon", "matrix")]


def deep_operator(pm, cls, inner, rng):
    """a window operator with tapertype=None and nover > nwin / 2 (four windows per sample along its window axes),
    traces / samples past the last window; returns (operator, inner operator, its float64 matrix, the Geo of the
    windows)"""
    L = pm.local
    nt = 12
    t = np.arange(nt) * 0.004
    three = cls.endswith("3D")
    ny, nx = (6, 8) if three else (1, 8)
    ns, ntw = (nt, nt) if cls.startswith("Sliding") else (19, 8)        # Patch: windows of 8 samples, step 2
    if inner == "radon":
        kind = "hyperbolic" if three else "parabolic"
        hs = [np.arange(ny) * 10.0, np.arange(nx) * 12.5]
        ps = [np.linspace(2000.0, 4000.0, 3), np.linspace(1500.0, 4000.0, 5)] if kind == "hyperbolic" else \
            [np.linspace(-1e-5, 1e-5, 3), np.linspace(-2e-5, 2e-5, 5)]
        tt = t[:ntw]
        Op = L.Radon3D(tt, *hs, *ps, kind=kind) if three else L.Radon2D(tt, hs[1], ps[1], kind=kind)
        ax = [host(a) for a in Op._axes]
        hy, hx, py, px = ax if three else (None, ax[0], None, ax[1])
        A = radon_sparse(kind, True, ntw, hx, px, hy, py)
        nop = tuple(Op.dims)
    else:
        A = sp.csr_matrix(rng.standard_normal((ny * nx * ntw, 7)))
        Op = L.MatrixMult(A.toarray())
        nop = (7,)
    n = (ny + 2 * 3 + 1 if three else 1, nx + 2 * 3 + 1, ns)
    if cls == "Sliding2D":
        nw, dims, _, _ = L.sliding2d_design((n[1], nt), nx, nx - 2, (Op.shape[1] // nt, nt) if inner == "radon"
                                            else (7, 1))
        S = L.Sliding2D(Op, dims, (n[1], nt), nx, nx - 2, tapertype=None)
        G = Geo("windows", "linear", True, None, np.zeros(nx), None, np.zeros(1), nt, n, (1, nw, 1), (1, 2, 1))
    elif cls == "Sliding3D":
        nopx = nop if inner == "radon" else (7, 1, 1)
        nw, dims, _, _ = L.sliding3d_design(n, (ny, nx), (ny - 2, nx - 2), nopx)
        S = L.Sliding3D(Op, dims, n, (ny, nx), (ny - 2, nx - 2), nopx, tapertype=None)
        G = Geo("windows", "linear", True, np.zeros(ny), np.zeros(nx), np.zeros(1), np.zeros(1), nt, n,
                (*nw, 1), (2, 2, 1))
    elif cls == "Patch2D":
        nopx = nop if inner == "radon" else (7, 1)
        nw, dims, _, _ = L.patch2d_design((n[1], ns), (nx, ntw), (nx - 2, ntw - 2), nopx)
        S = L.Patch2D(Op, dims, (n[1], ns), (nx, ntw), (nx - 2, ntw - 2), nopx, tapertype=None)
        G = Geo("patches", "linear", True, None, np.zeros(nx), None, np.zeros(1), ntw, n, (1, *nw), (1, 2, 2))
    else:
        nopx = nop if inner == "radon" else (7, 1, 1)
        nw, dims, _, _ = L.patch3d_design(n, (ny, nx, ntw), (ny - 2, nx - 2, ntw - 2), nopx)
        S = L.Patch3D(Op, dims, n, (ny, nx, ntw), (ny - 2, nx - 2, ntw - 2), nopx, tapertype=None)
        G = Geo("patches", "linear", True, np.zeros(ny), np.zeros(nx), np.zeros(1), np.zeros(1), ntw, n, nw,
                (2, 2, 2))
    assert G.depth() >= 3 ** (3 if cls == "Patch3D" else 2 if cls != "Sliding2D" else 1)
    return S, Op, A, G


@pytest.mark.gpu
@pytest.mark.parametrize("op", OPERATORS, ids=[f"{c}-{i}" for c, i in OPERATORS])
def test_deep_overlap_operators(pm, op):
    """Sliding2D / Sliding3D / Patch2D / Patch3D with four windows over a sample per window axis: against
    window_matrix of the inner operator's float64 matrix (bound), dottest, and (Radon) the fused apply against the
    generic per-window path bit for bit"""
    import torch
    from pylops_mpi_b200.utils.dottest import dottest
    cls, inner = op
    rng = np.random.default_rng(OPERATORS.index(op))
    S, Op, A, G = deep_operator(pm, cls, inner, rng)
    assert (S._fused is Op) == (inner == "radon")
    W = window_matrix(G, A, np.float64)
    assert W.shape == S.shape
    for adjoint in (False, True):
        x = rng.standard_normal(S.shape[0] if adjoint else S.shape[1])
        xt = torch.as_tensor(x).cuda()
        got = host(S.rmatvec(xt) if adjoint else S.matvec(xt))
        k = max_terms(A, adjoint)
        check_matrix(got[:, None], W.T.tocsr() if adjoint else W, x[:, None], k, 0 if adjoint else G.depth(),
                     np.float64, f"operator {cls}-{inner} {'adj' if adjoint else 'fwd'}")
        if inner == "radon":
            U = copy.copy(S)
            U._fused, U._work = None, {}
            for data in (xt, xt.float(), torch.complex(xt, torch.as_tensor(rng.standard_normal(x.size)).cuda())):
                a = S.rmatvec(data) if adjoint else S.matvec(data)
                b = U.rmatvec(data) if adjoint else U.matvec(data)
                assert torch.equal(a, b), f"{cls} adjoint={adjoint} {data.dtype}: fused != generic"
    B = pm.MPIBlockDiag([S])
    u = pm.DistributedArray.to_dist(rng.standard_normal(B.shape[1]))
    v = pm.DistributedArray.to_dist(rng.standard_normal(B.shape[0]))
    assert dottest(B, u, v, rtol=1e-12)
