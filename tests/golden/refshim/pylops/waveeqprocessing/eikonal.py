"""First-arrival traveltimes on a grid -- TEST INFRASTRUCTURE standing in for ``skfmm.travel_time``, which pylops 2.x's
``Kirchhoff(mode="eikonal")`` calls.  This is the one NumPy statement of the discrete problem that
``b2_eikonal_tables`` (pylops_mpi_b200/csrc/eikonal.cu) solves; the device tables equal it bit for bit.

The scheme: T = 0 at the point's node, +inf elsewhere, then Jacobi steps of the first-order Godunov upwind update
until a step changes no value (or ``max_iter`` steps).  Per node, from the previous iterate only: ``s = 1 / vel``;
``a_k`` the smaller of the two neighbours along axis k (+inf off the grid); the (a_k, h_k, w_k = 1 / (h_k * h_k))
stably sorted by a_k (ties keep y, x, z order); ``t = a1 + h1 * s``; while a next axis exists and ``t > a_next``,
``t`` becomes the larger root of ``sum_k w_k (t - a_k)**2 = s**2`` over the axes used, written relative to a1 with
``d_k = a_k - a1``, ``p_k = w_k * d_k``, ``q_k = p_k * d_k``: ``A = sum w``, ``B = sum p``, ``C = sum q - s * s``,
``t = a1 + (B + sqrt(max(B * B - A * C, 0))) / A`` (sums left to right); new value ``min(old, t)``.

Differences from scikit-fmm (what pylops uses): it is first order everywhere and puts T = 0 on the source node,
where scikit-fmm with its default ``order=2`` uses second-order differences where it can and places the zero level
set half a cell from the node.  Tables differ from pylops + scikit-fmm by O(h / v), most near the source."""
import numpy as np


def godunov_step(T, slow, h, w):
    """one Jacobi step: the updated copy of T (..., ny, nx, nz); slow (ny, nx, nz), h and w per axis (y, x, z)"""
    pad = [(0, 0)] * (T.ndim - 3) + [(1, 1)] * 3
    P = np.pad(T, pad, constant_values=np.inf)

    def nb(axis):
        """the smaller of the two neighbours along spatial axis 0, 1, 2 (y, x, z)"""
        lo, hi = [slice(1, -1)] * 3, [slice(1, -1)] * 3
        lo[axis], hi[axis] = slice(None, -2), slice(2, None)
        return np.minimum(P[(Ellipsis, *lo)], P[(Ellipsis, *hi)])

    A = np.stack((nb(0), nb(1), nb(2)), axis=-1)
    order = np.argsort(A, axis=-1, kind="stable")
    a = np.take_along_axis(A, order, axis=-1)
    hh, ww = np.asarray(h, dtype=np.float64)[order], np.asarray(w, dtype=np.float64)[order]
    a1, a2, a3 = a[..., 0], a[..., 1], a[..., 2]
    h1, w1, w2, w3 = hh[..., 0], ww[..., 0], ww[..., 1], ww[..., 2]
    s = np.broadcast_to(slow, T.shape)
    t = a1 + h1 * s
    with np.errstate(invalid="ignore", over="ignore"):
        sq = s * s
        d2 = a2 - a1
        p2 = w2 * d2
        q2 = p2 * d2
        A2 = w1 + w2
        t2 = a1 + (p2 + np.sqrt(np.maximum(p2 * p2 - A2 * (q2 - sq), 0.0))) / A2
        t = np.where(t > a2, t2, t)
        d3 = a3 - a1
        p3 = w3 * d3
        q3 = p3 * d3
        A3, B3 = A2 + w3, p2 + p3
        t3 = a1 + (B3 + np.sqrt(np.maximum(B3 * B3 - A3 * ((q2 + q3) - sq), 0.0))) / A3
        t = np.where(t > a3, t3, t)
    return np.minimum(T, t)


def jacobi(vel, spacing, nodes, max_iter=None):
    """(T, iters): the traveltime fields (n, ny, nx, nz) from ``nodes`` (n, 3) integer (iy, ix, iz) through ``vel``
    (ny, nx, nz), spacings ``(dy, dx, dz)``; ``iters`` is the number of Jacobi steps that changed a value.  With
    ``max_iter``, T is the iterate after at most that many steps (the fixed point if reached by then)."""
    vel = np.asarray(vel, dtype=np.float64)
    h = np.asarray(spacing, dtype=np.float64)
    w = 1.0 / (h * h)
    slow = 1.0 / vel
    nodes = np.asarray(nodes, dtype=np.int64).reshape(-1, 3)
    T = np.full((len(nodes),) + vel.shape, np.inf)
    T[np.arange(len(nodes)), nodes[:, 0], nodes[:, 1], nodes[:, 2]] = 0.0
    it = 0
    while max_iter is None or it < max_iter:
        N = godunov_step(T, slow, h, w)
        if np.array_equal(N, T):
            break
        T = N
        it += 1
    return T, it


def snap(pts, axes):
    """grid nodes (n, 3) of points (ndim, n) with rows ((y,) x, z) on uniform axes ((y,) x, z): per axis
    ``round((p - axis[0]) / d)`` with NumPy's half-to-even rounding, as pylops' eikonal branch computes them
    (a 2-D point gets iy = 0)"""
    pts = np.asarray(pts, dtype=np.float64)
    cols = []
    for p, a in zip(pts, axes):
        a = np.asarray(a, dtype=np.float64)
        d = a[1] - a[0] if a.size > 1 else 1.0
        cols.append(np.round((p - a[0]) / d).astype(np.int64))
    if len(cols) == 2:
        cols.insert(0, np.zeros_like(cols[0]))
    return np.stack(cols, axis=1)


def spacings(axes):
    """(dy, dx, dz) of uniform axes ((y,) x, z); a one-point axis and a missing y get 1.0"""
    d = [float(a[1] - a[0]) if np.asarray(a).size > 1 else 1.0 for a in axes]
    return tuple([1.0] * (3 - len(d)) + d)


def traveltime_table(vel, axes, pts):
    """the (ni, n) float64 table of pylops' layout (ii = ix * nz + iz, 3-D (iy * nx + ix) * nz + iz) for points
    ``pts`` (ndim, n) through ``vel`` of the image shape on the uniform ``axes`` ((y,) x, z)"""
    vel = np.asarray(vel, dtype=np.float64)
    v3 = vel.reshape((1,) * (3 - vel.ndim) + vel.shape)
    T, _ = jacobi(v3, spacings(axes), snap(pts, axes))
    return T.reshape(T.shape[0], -1).T.copy()
