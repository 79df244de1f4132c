"""The float64 definition of the non-stationary convolutions and filter estimation (NonStationaryConvolve2D / 3D,
NonStationaryFilters1D / 2D), and the checks of their kernels through the C ABI, shared by test_nsconvolve2d.py,
test_nsconvolve3d.py and test_nsfilters.py.

    h_j = sum_c dt(prod_d w_(c_d)(j_d)) hs[c]     (the product from the last axis to the first, rounded once)
    forward y[i] = sum_j h_j[hc + i - j] x[j],  adjoint the transpose

with per axis, v = (j - oh) / dh: weight 1 on the end filter outside the nodes, else 1 - (v - l) on l = floor(v) and
v - l on l + 1."""
import itertools

import numpy as np

from op_checks import guarded_twice

U = {np.float32: 2.0 ** -24, np.float64: 2.0 ** -53}


def axis_weights(j, oh, dh, nf):
    """{filter: float64 weight} of sample j by the definition: weight 1 on the end filter outside the nodes"""
    v = (j - oh) / dh
    lo = int(np.floor(v))
    if lo < 0:
        return {0: 1.0}
    if lo >= nf - 1:
        return {nf - 1: 1.0}
    w = v - lo
    return {lo: 1.0 - w, lo + 1: w} if w != 0.0 else {lo: 1.0}


def axis_w(n, oh, dh, nf):
    """(nf, n) float64 weights of every sample on every filter"""
    W = np.zeros((nf, n))
    for j in range(n):
        for a, w in axis_weights(j, oh, dh, nf).items():
            W[a, j] = w
    return W


def point_weights(j, oh, dh, nf, dt):
    """[(c, W_c)] of point j, one entry per axis in j, oh, dh and nf: W = dt(w_z * ... * w_x), from the last axis"""
    ws = [axis_weights(*a) for a in zip(j, oh, dh, nf)]
    out = []
    for c in itertools.product(*ws):
        W = ws[-1][c[-1]]
        for d in range(len(ws) - 2, -1, -1):
            W = W * ws[d][c[d]]
        out.append((c, float(dt(W))))
    return out


def ns_matrix(hs, dims, oh, dh, absolute=False):
    """M[i, j] = h_j[hc + i - j] in float64 for a bank hs of shape nf + nh on a ``dims`` block, h_j = sum W_c hs[c]
    with W rounded to the dtype of hs (absolute: sum W_c |hs[c]|, the magnitude of the terms)"""
    nd = len(dims)
    nf, nh = hs.shape[:nd], hs.shape[nd:]
    hc = tuple(n // 2 for n in nh)
    h64 = np.abs(hs.astype(np.float64)) if absolute else hs.astype(np.float64)
    M = np.zeros(tuple(dims) * 2)
    for j in np.ndindex(*dims):
        h = sum(W * h64[c] for c, W in point_weights(j, oh, dh, nf, hs.dtype.type))
        lo = [max(0, j[d] - hc[d]) for d in range(nd)]
        hi = [min(dims[d], j[d] + hc[d] + 1) for d in range(nd)]
        M[tuple(slice(a, b) for a, b in zip(lo, hi)) + j] = \
            h[tuple(slice(lo[d] - j[d] + hc[d], hi[d] - j[d] + hc[d]) for d in range(nd))]
    n = int(np.prod(dims))
    return M.reshape(n, n)


def gamma(n, dt):
    """gamma_n = n u / (1 - n u): the relative bound of a chain of n rounded operations in dtype dt"""
    return n * U[dt] / (1 - n * U[dt])


def assert_within(got, ref, tol):
    """componentwise |got - ref| <= tol"""
    err = np.abs(got.reshape(ref.shape).astype(np.float64) - ref)
    assert np.all(err <= tol), f"max err {err.max():.3e}, excess {(err - tol).max():.3e}"


_MATRICES = {}


def reference(x, hs, oh, dh, adjoint, dt):
    """(float64 product of the definition, gamma_n sum |terms|) for x (dims[, ni]) and a bank of d-D filters, n the
    number of rounded operations in one output's longest chain: 2^d nh_1 ... nh_d fma (each point takes up to 2^d
    filters), a weight and a product per term"""
    nd = hs.ndim // 2
    dims = x.shape[:nd]
    key = (hs.astype(dt).tobytes(), hs.shape, dims, oh, dh)
    if key not in _MATRICES:
        _MATRICES.clear()
        _MATRICES[key] = tuple(ns_matrix(hs.astype(dt), dims, oh, dh, absolute=a) for a in (False, True))
    M, B = _MATRICES[key]
    M, B = (M.T, B.T) if adjoint else (M, B)
    xs = x.reshape(int(np.prod(dims)), -1).astype(np.float64)
    n = 2 ** nd * int(np.prod(hs.shape[nd:])) + 4 * nd
    return M @ xs, gamma(n, dt) * (B @ np.abs(xs))


def check_close(got, x, hs, oh, dh, adjoint, dt):
    """componentwise |got - ref| <= gamma_n (sum |terms|) against the float64 product of the definition"""
    ref, tol = reference(x, hs, oh, dh, adjoint, dt)
    assert_within(got, ref, tol)


# ---------------------------------------------------------------------------------------------------------------
# the kernels through the C ABI
# ---------------------------------------------------------------------------------------------------------------
def c_ns(pm, x, y, dims, ni, hs, nf, nh, oh, dh, adjoint, code):
    """b2_nsconvolve2d / b2_nsconvolve3d, by the rank of ``dims``"""
    L = pm._lib
    fn = L.lib.b2_nsconvolve2d if len(dims) == 2 else L.lib.b2_nsconvolve3d
    return fn(L.ctx(), x, y, *dims, ni, hs, *nf, *nh, *(v for od in zip(oh, dh) for v in od), adjoint, code,
              L.stream())


def run_kernel(pm, x_np, hs_np, oh, dh, adjoint, dt, guard=5):
    """apply the d-D bank hs_np to x_np (dims[, 2]) through the C ABI into a guarded interior view; returns (y, guards
    intact, second apply bit-equal)"""
    import torch
    nd = hs_np.ndim // 2
    x = torch.as_tensor(np.ascontiguousarray(x_np.ravel(), dtype=dt)).cuda()
    hs = torch.as_tensor(np.ascontiguousarray(hs_np, dtype=dt)).cuda()
    ni = x_np.shape[nd] if x_np.ndim == nd + 1 else 1
    code = pm._lib.F32 if dt == np.float32 else pm._lib.F64
    y, guards_ok, same = guarded_twice(
        lambda yp: c_ns(pm, x.data_ptr(), yp, x_np.shape[:nd], ni, hs.data_ptr(), hs_np.shape[:nd], hs_np.shape[nd:],
                        oh, dh, int(adjoint), code), x_np.size, dt, guard)
    return y.reshape(x_np.shape), guards_ok, same


# ---------------------------------------------------------------------------------------------------------------
# the definition at chosen outputs, without a dense matrix
# ---------------------------------------------------------------------------------------------------------------
class Geometry(tuple):
    """(dims, nf, nh, oh, dh), one entry per axis in each"""

    def __new__(cls, dims, nf, nh, oh, dh):
        return super().__new__(cls, tuple(tuple(int(v) for v in t) for t in (dims, nf, nh, oh, dh)))

    dims, nf, nh, oh, dh = (property(lambda s, k=k: s[k]) for k in range(5))
    hc = property(lambda s: tuple(n // 2 for n in s.nh))
    nd = property(lambda s: len(s.dims))


def axis_at(j, oh, dh, nf):
    """(first filter, (B, 2) float64 weights on it and the next) of each sample of the integer array j, from
    point_weights on the distinct samples"""
    u, inv = np.unique(np.asarray(j, dtype=np.int64), return_inverse=True)
    f0, w = np.zeros(len(u), np.int64), np.zeros((len(u), 2))
    for i, jj in enumerate(u):
        ws = sorted(point_weights((int(jj),), (oh,), (dh,), (nf,), np.float64))
        f0[i] = ws[0][0][0]
        for m, (_, W) in enumerate(ws):
            w[i, m] = W
    inv = inv.reshape(np.shape(j))
    return f0[inv], w[inv]


def _taps(g, hs, wc, kk, dt, magnitude=True):
    """(h, |h|) with h[b, k] = sum_c dt(W_c(j)) hs[c][k] (float64), j = (wc[0][b, k_0], wc[1][b, k_1], ...) per axis
    and the taps k = (kk[0][b, k_0], ...); the weight product is point_weights', from the last axis to the first
    (|h| = sum_c |W_c hs[c][k]|, or None without ``magnitude``)"""
    nd, B = g.nd, wc[0].shape[0]
    tabs = [axis_at(np.clip(wc[d], 0, g.dims[d] - 1), g.oh[d], g.dh[d], g.nf[d]) for d in range(nd)]

    def bcast(a, d):                    # (B, n_d) -> (B, 1, .., n_d, .., 1)
        shape = [B] + [1] * nd
        shape[1 + d] = a.shape[1]
        return a.reshape(shape)

    h, ha = 0.0, (0.0 if magnitude else None)
    hsf = hs.astype(np.float64).ravel()
    tap = 0
    for d in range(nd):
        tap = tap * g.nh[d] + bcast(kk[d], d)
    for bits in itertools.product((0, 1), repeat=nd):
        W, fidx = None, 0
        for d in range(nd - 1, -1, -1):
            wd = bcast(tabs[d][1][..., bits[d]], d)
            W = wd if W is None else W * wd
        if dt != np.float64:
            W = W.astype(dt).astype(np.float64)
        for d in range(nd):
            fidx = fidx * g.nf[d] + bcast(np.minimum(tabs[d][0] + bits[d], g.nf[d] - 1), d)
        hv = hsf[fidx * int(np.prod(g.nh)) + tap]
        h = h + W * hv
        if magnitude:
            ha = ha + np.abs(W * hv)
    return h, ha


def _read(x, coords, dims):
    """x at the integer coordinates (one broadcastable array per axis), 0 outside dims: (..., n_inner); x is an
    array (dims[, n_inner]) or a callable of the coordinates returning (..., n_inner)"""
    inside = np.ones(np.broadcast(*coords).shape, bool)
    for c, n in zip(coords, dims):
        inside &= (c >= 0) & (c < n)
    cl = [np.clip(c, 0, n - 1) for c, n in zip(coords, dims)]
    if callable(x):
        v = x(*np.broadcast_arrays(*cl))
    else:
        v = x[tuple(cl)]
        if x.ndim == len(dims):
            v = v[..., None]
    return np.where(inside[..., None], v.astype(np.float64), 0.0)


def nterms(g):
    """the rounded operations in one output's longest chain (reference's n)"""
    return 2 ** g.nd * int(np.prod(g.nh)) + 4 * g.nd


def point_ref(g, hs, x, outs, adjoint, dt, batch=None, bound=True):
    """(value, sum |terms|) of the definition in float64 at the outputs ``outs`` (B, nd), each (B, n_inner), summed
    over each output's footprint:  forward y[i] = sum_k h_(i + hc - k)[k] x[i + hc - k], adjoint
    x[j] = sum_k h_j[k] y[j + k - hc]; h_j from point_weights, its weight product rounded to dt (without
    ``bound`` the second is None)"""
    outs = np.asarray(outs, np.int64)
    K = int(np.prod(g.nh))
    batch = batch or max(1, 2_000_000 // K)
    vals, bnds = [], []
    for s in range(0, len(outs), batch):
        o = outs[s:s + batch]
        kk = [np.broadcast_to(np.arange(g.nh[d]), (len(o), g.nh[d])) for d in range(g.nd)]
        if adjoint:
            wc = [np.broadcast_to(o[:, d:d + 1], (len(o), g.nh[d])) for d in range(g.nd)]
            dc = [o[:, d:d + 1] + kk[d] - g.hc[d] for d in range(g.nd)]
        else:
            wc = dc = [o[:, d:d + 1] + g.hc[d] - kk[d] for d in range(g.nd)]
        h, ha = _taps(g, hs, wc, kk, dt, magnitude=bound)
        shp = [len(o)] + [1] * g.nd
        inside = np.ones(h.shape, bool)
        for d in range(g.nd):       # the weight's sample must lie in the image too (forward: it is the data's)
            s_ = list(shp)
            s_[1 + d] = g.nh[d]
            inside &= ((wc[d] >= 0) & (wc[d] < g.dims[d])).reshape(s_)
        coords = []
        for d in range(g.nd):
            s_ = list(shp)
            s_[1 + d] = g.nh[d]
            coords.append(dc[d].reshape(s_))
        v = _read(x, coords, g.dims) * inside[..., None]
        ax = tuple(range(1, g.nd + 1))
        vals.append(np.sum(h[..., None] * v, axis=ax))
        if bound:
            bnds.append(np.sum(ha[..., None] * np.abs(v), axis=ax))
    return np.concatenate(vals), (np.concatenate(bnds) if bound else None)


def spike_ref(g, hs, pos, val, adjoint, dt, n_inner=1):
    """the whole float64 output (dims, n_inner) for an input that is zero except val (P, n_inner) at the samples pos
    (P, nd): each spike adds its interpolated filter (forward) or the transposed footprint (adjoint)"""
    pos = np.asarray(pos, np.int64)
    val = np.asarray(val, np.float64).reshape(len(pos), n_inner)
    out = np.zeros(g.dims + (n_inner,))
    K = int(np.prod(g.nh))
    batch = max(1, 2_000_000 // K)
    for s in range(0, len(pos), batch):
        p, v = pos[s:s + batch], val[s:s + batch]
        kk = [np.broadcast_to(np.arange(g.nh[d]), (len(p), g.nh[d])) for d in range(g.nd)]
        if adjoint:         # spike at i reaches j = i + hc - k with tap k of h_j
            wc = oc = [p[:, d:d + 1] + g.hc[d] - kk[d] for d in range(g.nd)]
        else:               # spike at j reaches i = j + k - hc with tap k of h_j
            wc = [np.broadcast_to(p[:, d:d + 1], (len(p), g.nh[d])) for d in range(g.nd)]
            oc = [p[:, d:d + 1] + kk[d] - g.hc[d] for d in range(g.nd)]
        h, _ = _taps(g, hs, wc, kk, dt, magnitude=False)
        shp = [len(p)] + [1] * g.nd
        full = []
        for d in range(g.nd):
            s_ = list(shp)
            s_[1 + d] = g.nh[d]
            full.append(np.broadcast_to(oc[d].reshape(s_), h.shape))
        inside = np.ones(h.shape, bool)
        for d in range(g.nd):
            inside &= (full[d] >= 0) & (full[d] < g.dims[d])
        terms = h[..., None] * v.reshape([len(p)] + [1] * g.nd + [n_inner])
        np.add.at(out, tuple(f[inside] for f in full), terms[inside])
    return out


def filter_window(n, oh, dh, nf, a):
    """samples that may carry a weight of filter a: [node a - 1, node a + 1], to the edge for the end filters (the
    weights from point_weights decide which of them do)"""
    lo = 0 if a == 0 else oh + (a - 1) * dh
    hi = n if a == nf - 1 else oh + (a + 1) * dh + 1
    return max(lo, 0), min(hi, n)


def nsfilters_ref(g, d, inp, taps, dt):
    """(value, sum |terms|, terms) of g_c[k] = sum_(j in S_c) W_c[j] inp[j] d[j + k - hc] in float64 at the bank
    entries ``taps`` (B, 4) = (a, b, kx, kz), each one dot product over the filter's support (W_c rounded to dt; d
    and inp arrays (nx, nz) or callables of (jx, jz)); terms counts the support's samples"""
    taps = np.asarray(taps, np.int64)
    val, bnd, nt = np.zeros(len(taps)), np.zeros(len(taps)), np.zeros(len(taps), np.int64)
    for c in {(int(a), int(b)) for a, b in taps[:, :2]}:
        xl, xh = filter_window(g.dims[0], g.oh[0], g.dh[0], g.nf[0], c[0])
        zl, zh = filter_window(g.dims[1], g.oh[1], g.dh[1], g.nf[1], c[1])
        jx, jz = np.arange(xl, xh), np.arange(zl, zh)
        fx, wx = axis_at(jx, g.oh[0], g.dh[0], g.nf[0])
        fz, wz = axis_at(jz, g.oh[1], g.dh[1], g.nf[1])
        wx = np.where(fx == c[0], wx[:, 0], np.where(fx + 1 == c[0], wx[:, 1], 0.0))
        wz = np.where(fz == c[1], wz[:, 0], np.where(fz + 1 == c[1], wz[:, 1], 0.0))
        jx, wx, jz, wz = jx[wx != 0], wx[wx != 0], jz[wz != 0], wz[wz != 0]
        W = (wz[None, :] * wx[:, None]).astype(dt).astype(np.float64)
        u = W * _read(inp, (jx[:, None], jz[None, :]), g.dims)[..., 0]
        nz = np.nonzero(u)
        ux, uz, uv = jx[nz[0]], jz[nz[1]], u[nz]
        sel = np.nonzero((taps[:, 0] == c[0]) & (taps[:, 1] == c[1]))[0]
        for s in range(0, len(sel), max(1, 4_000_000 // max(len(uv), 1))):
            i = sel[s:s + max(1, 4_000_000 // max(len(uv), 1))]
            dv = _read(d, (ux[None, :] + taps[i, 2:3] - g.hc[0], uz[None, :] + taps[i, 3:4] - g.hc[1]),
                       g.dims)[..., 0]
            val[i] = np.sum(uv[None, :] * dv, axis=1)
            bnd[i] = np.sum(np.abs(uv[None, :] * dv), axis=1)
        nt[sel] = len(jx) * len(jz)
    return val, bnd, nt


def tile_sizes(nd, dt, adjoint):
    """outputs per CTA along each axis: 32 x 64 in 2-D; TX x 32 x 64 in 3-D, TX = 4 / 2 (float32 forward /
    adjoint) and 1 (float64)"""
    if nd == 2:
        return (32, 64)
    return (1 if dt == np.float64 else 2 if adjoint else 4, 32, 64)


def axis_specials(n, T, oh, dh, nf):
    """the samples of one axis worth checking: both sides of every tile seam, every node and its neighbours (a
    support's edges are the neighbouring nodes +- 1) and the first and last two samples"""
    s = set()
    for m in range(T, n, T):
        s |= {m - 1, m}
    for a in range(-1, nf + 1):
        s |= {oh + a * dh + e for e in (-1, 0, 1)}
    s |= {0, 1, n - 2, n - 1}
    return np.array(sorted(v for v in s if 0 <= v < n), np.int64)


def seam_outputs(g, dt, adjoint, need=2048, seed=0):
    """(B, nd) outputs worth checking, at least ``need`` (or every output): each axis's special samples, each once
    with random special or plain samples on the other axes, then random fill"""
    rng = np.random.default_rng(seed)
    T = tile_sizes(g.nd, dt, adjoint)
    sp = [axis_specials(n, t, o, h, f) for n, t, o, h, f in zip(g.dims, T, g.oh, g.dh, g.nf)]
    total = int(np.prod(g.dims))
    if total <= need:
        return np.stack(np.unravel_index(np.arange(total), g.dims), 1).astype(np.int64)
    pts = []
    for d in range(g.nd):
        for v in sp[d]:
            p = [rng.choice(sp[e]) if rng.random() < 0.5 else rng.integers(g.dims[e]) for e in range(g.nd)]
            p[d] = v
            pts.append(p)
    pts = np.unique(np.array(pts, np.int64), axis=0)
    while len(pts) < need:
        extra = np.stack([rng.integers(0, n, need) for n in g.dims], 1)
        pts = np.unique(np.concatenate([pts, extra]), axis=0)
    return pts
