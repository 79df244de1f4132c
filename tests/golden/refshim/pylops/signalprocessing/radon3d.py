"""Restatement of third-party ``pylops.signalprocessing.Radon3D`` (pylops 2.x, as remembered) -- TEST
INFRASTRUCTURE for tests/golden/make_golden_radon.py.  Radon2D's restatement (radon2d.py) with a y axis: the traces
are the (hy, hx) grid, y outer, the model traces the (py, px) grid, y outer, and the y term is added last
(remembered term order): ``(t0 + px*hx) + py*hy``, ``(t0 + px*hx**2) + py*hy**2``,
``sqrt((t0**2 + (hx/px)**2) + (hy/py)**2)``."""
import numpy as np

from .radon2d import _Spread, _check, _create_table, _unitless


def _linear(y, x, t, py, px):
    return t + px * x + py * y


def _parabolic(y, x, t, py, px):
    return t + px * x ** 2 + py * y ** 2


def _hyperbolic(y, x, t, py, px):
    return np.sqrt(t ** 2 + (x / px) ** 2 + (y / py) ** 2)


CURVES = {"linear": _linear, "parabolic": _parabolic, "hyperbolic": _hyperbolic}


class Radon3D(_Spread):
    """Radon3D(taxis, hyaxis, hxaxis, pyaxis, pxaxis, kind, centeredh, interp, onthefly, engine, dtype, name): model
    (npy, npx, nt), data (nhy, nhx, nt)"""

    def __init__(self, taxis, hyaxis, hxaxis, pyaxis, pxaxis, kind="linear", centeredh=True, interp=True,
                 onthefly=False, engine="numpy", dtype="float64", name="R"):
        _check(kind, engine, dtype)
        hy, py, _, _ = _unitless(taxis, hyaxis, pyaxis, kind, centeredh, "hyaxis")
        hx, px, _, _ = _unitless(taxis, hxaxis, pxaxis, kind, centeredh, "hxaxis")
        nt = np.asarray(taxis).size
        HY, HX = (a.ravel() for a in np.meshgrid(hy, hx, indexing="ij"))
        PY, PX = (a.ravel() for a in np.meshgrid(py, px, indexing="ij"))
        f = CURVES[kind]
        table, dtable = _create_table(lambda ip, it: f(HY, HX, it, PY[ip], PX[ip]), PY.size, nt, HY.size, interp)
        self.kind, self.engine, self.onthefly = kind, engine, onthefly
        super().__init__(table, dtable, (py.size, px.size, nt), (hy.size, hx.size, nt), interp, dtype, name)
