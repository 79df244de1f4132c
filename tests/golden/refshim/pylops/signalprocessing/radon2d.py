"""Restatement of third-party ``pylops.signalprocessing.Radon2D`` (pylops 2.x, as remembered: pylops is not
installed here to check it) -- TEST INFRASTRUCTURE so that the reference's MPIBlockDiag and FISTA can be run over
rank-local sparse Radon transforms of CMP gathers by tests/golden/make_golden_radon.py.

It follows pylops' structure: the axes are made unitless (``_unitless``), ``_indices_2d`` gives the index and weight
of every (model sample, trace) pair, ``_create_table`` stores them per model sample (NaN where the mask drops the
pair), and ``Spread``'s loops apply them (model samples in (t0, p) order).  Remembered items: the centred offsets
``arange(nh) - nh // 2 + ((nh + 1) % 2) / 2``, the unit factors of ``p`` per kind (``dh / dt``, ``dh**2 / dt``,
``dt / dh``; ``**2`` is ``x*x``), the mask ``0 <= tdec < nt - 1`` (``nt`` without interpolation) and ``np.fix`` for
the index.

Sums are float64 (complex128 for complex data) and rounded once to the result dtype, where pylops' numpy engine adds
into an array of the operator's dtype; the adjoint adds ``x[it] * (1 - d) + x[it + 1] * d`` per trace in trace order,
where pylops sums each tap over the traces with ``np.sum``.  Neither changes a result on exactly representable data.
"""
import numpy as np

from .. import LinearOperator

KINDS = ("linear", "parabolic", "hyperbolic")


def _linear(x, t, px):
    return t + px * x


def _parabolic(x, t, px):
    return t + px * x ** 2


def _hyperbolic(x, t, px):
    return np.sqrt(t ** 2 + (x / px) ** 2)


CURVES = {"linear": _linear, "parabolic": _parabolic, "hyperbolic": _hyperbolic}


def _sampling(name, axis):
    if axis.size < 2:
        raise ValueError(f"{name} needs at least 2 samples to define its sampling")
    return np.abs(axis[1] - axis[0])


def _unitless(taxis, haxis, paxis, kind, centeredh, hname="haxis"):
    """(h, p, dt, dh): offsets in samples of dh and slownesses (velocities for hyperbolic) in samples per trace"""
    taxis, haxis, paxis = (np.asarray(a, dtype=np.float64).ravel() for a in (taxis, haxis, paxis))
    dt, dh = _sampling("taxis", taxis), _sampling(hname, haxis)
    nh = haxis.size
    h = np.arange(nh) - nh // 2 + ((nh + 1) % 2) / 2 if centeredh else haxis / dh
    if kind == "linear":
        p = paxis * (dh / dt)
    elif kind == "parabolic":
        p = paxis * (dh * dh / dt)          # dh**2, pinned to x*x as NumPy squares arrays
    else:
        p = paxis * (dt / dh)
    return h, p, dt, dh


def _check(kind, engine, dtype):
    if engine not in ("numpy", "numba", "cuda"):
        raise KeyError("engine must be numpy or numba or cuda")
    if kind not in KINDS:
        raise NotImplementedError(f"kind {kind} is not supported")
    if np.iscomplexobj(np.ones(1, dtype=dtype)):
        raise NotImplementedError(f"dtype {dtype} is not supported")


def _indices_2d(tdecscan, nt, interp=True):
    """pylops' mask, index and weight of the pairs of one model sample: (used, it, d)"""
    if not interp:
        xscan = (tdecscan >= 0) & (tdecscan < nt)
    else:
        xscan = (tdecscan >= 0) & (tdecscan < nt - 1)
    tscanfs = np.fix(tdecscan[xscan]).astype(int)
    dtscan = tdecscan[xscan] - tscanfs if interp else None
    return xscan, tscanfs, dtscan


def _create_table(tdec_of, npm, nt, nh, interp):
    """table[ip, it, ih] = sample index of the pair (NaN if dropped), dtable its weight d"""
    table = np.full((npm, nt, nh), np.nan)
    dtable = np.full((npm, nt, nh), np.nan) if interp else None
    with np.errstate(divide="ignore", invalid="ignore"):
        for ip in range(npm):
            for it in range(nt):
                xscan, tscan, dtscan = _indices_2d(tdec_of(ip, it), nt, interp)
                table[ip, it, xscan] = tscan
                if interp:
                    dtable[ip, it, xscan] = dtscan
    return table, dtable


class _Spread(LinearOperator):
    """pylops' Spread over a (model trace, t0) -> (trace, sample) table; model (npm, nt), data (nh, nt) flattened"""

    def __init__(self, table, dtable, dims, dimsd, interp, dtype, name):
        self.table, self.dtable, self.interp = table, dtable, interp
        self.dims, self.dimsd = tuple(dims), tuple(dimsd)
        self.name = name
        super().__init__(dtype=np.dtype(dtype), shape=(int(np.prod(dimsd)), int(np.prod(dims))))

    def _out(self, x):
        return np.result_type(self.dtype, x.dtype)

    def _matvec(self, x):
        npm, nt, nh = self.table.shape
        x = np.asarray(x).reshape(npm, nt)
        y = np.zeros((nh, nt), dtype=np.result_type(np.float64, x.dtype))
        for it in range(nt):
            for ip in range(npm):
                indices = self.table[ip, it]
                mask = np.argwhere(~np.isnan(indices)).ravel()
                if mask.size > 0:
                    idx = indices[mask].astype(int)
                    if not self.interp:
                        y[mask, idx] += x[ip, it]
                    else:
                        d = self.dtable[ip, it, mask]
                        y[mask, idx] += (1 - d) * x[ip, it]
                        y[mask, idx + 1] += d * x[ip, it]
        return y.astype(self._out(x)).ravel()

    def _rmatvec(self, x):
        npm, nt, nh = self.table.shape
        x = np.asarray(x).reshape(nh, nt)
        y = np.zeros((npm, nt), dtype=np.result_type(np.float64, x.dtype))
        for it in range(nt):
            for ip in range(npm):
                indices = self.table[ip, it]
                mask = np.argwhere(~np.isnan(indices)).ravel()
                if mask.size > 0:
                    idx = indices[mask].astype(int)
                    if not self.interp:
                        terms = x[mask, idx]
                    else:
                        d = self.dtable[ip, it, mask]
                        terms = x[mask, idx] * (1 - d) + x[mask, idx + 1] * d
                    y[ip, it] = np.cumsum(terms)[-1]           # added one trace at a time, in trace order
        return y.astype(self._out(x)).ravel()


class Radon2D(_Spread):
    """Radon2D(taxis, haxis, pxaxis, kind, centeredh, interp, onthefly, engine, dtype, name): model (npx, nt), data
    (nh, nt); ``onthefly`` and ``engine`` do not change the values"""

    def __init__(self, taxis, haxis, pxaxis, kind="linear", centeredh=True, interp=True, onthefly=False,
                 engine="numpy", dtype="float64", name="R"):
        _check(kind, engine, dtype)
        h, p, _, _ = _unitless(taxis, haxis, pxaxis, kind, centeredh)
        nt = np.asarray(taxis).size
        f = CURVES[kind]
        table, dtable = _create_table(lambda ip, it: f(h, it, p[ip]), p.size, nt, h.size, interp)
        self.kind, self.engine, self.onthefly = kind, engine, onthefly
        super().__init__(table, dtable, (p.size, nt), (h.size, nt), interp, dtype, name)
