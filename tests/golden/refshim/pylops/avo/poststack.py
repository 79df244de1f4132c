"""Restatement of third-party ``pylops.avo.poststack.PoststackLinearModelling`` -- TEST INFRASTRUCTURE for
tests/golden/make_golden_poststack.py (imported as ``pylops.avo.poststack``)."""
import numpy as np

from .._algebra import ProductLinearOperator
from .._derivatives import FirstDerivative
from ..signalprocessing.convolve1d import Convolve1D


def PoststackLinearModelling(wav, nt0, spatdims=None, explicit=False, sparse=False, kind="centered"):
    """Restatement of third-party ``pylops.avo.poststack.PoststackLinearModelling`` (pylops 2.x, stationary real
    wavelet, matrix-free) -- TEST INFRASTRUCTURE so that the reference's MPIBlockDiag and solvers can be run over
    the post-stack modelling of tutorials/poststack.py.  As pylops builds it: ``dims = (nt0,) + spatdims`` and
    ``Convolve1D(dims, h=wav, offset=len(wav) // 2, axis=0) * FirstDerivative(dims, axis=0, sampling=1.0,
    kind=kind)``, with the operator dtype ``wav.dtype``."""
    wav = np.asarray(wav)
    if explicit or sparse or wav.ndim != 1 or np.iscomplexobj(wav):
        raise NotImplementedError("only the matrix-free operator with a stationary real wavelet is restated")
    if kind not in ("forward", "centered"):
        raise NotImplementedError(f"{kind} not an available derivative kind...")
    if spatdims is None:
        dims = (nt0,)
    elif np.ndim(spatdims) == 0:
        dims = (nt0, spatdims)
    else:
        dims = (nt0,) + tuple(spatdims)
    Cop = Convolve1D(dims, h=wav, offset=len(wav) // 2, axis=0, dtype=wav.dtype)
    Dop = FirstDerivative(dims, axis=0, sampling=1.0, kind=kind, dtype=wav.dtype)
    return ProductLinearOperator(Cop, Dop)             # pylops' Cop * Dop
