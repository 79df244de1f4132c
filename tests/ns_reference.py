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
