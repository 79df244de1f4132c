"""Restatement of third-party ``pylops.avo.poststack.PoststackLinearModelling`` including its 2-D (non-stationary)
wavelet branch -- TEST INFRASTRUCTURE for tests/golden/make_golden_nsconvolve.py.  A 1-D wavelet goes to the
stationary restatement (refshim/pylops/avo/poststack.py), unchanged."""
import numpy as np

from .._algebra import ProductLinearOperator
from .._derivatives import FirstDerivative
from ..basicoperators.matrixmult import MatrixMult
from ..utils.signalprocessing import nonstationary_convmtx
from . import poststack


def PoststackLinearModelling(wav, nt0, spatdims=None, explicit=False, sparse=False, kind="centered"):
    """pylops 2.x ``PoststackLinearModelling`` (matrix-free, real wavelet).  A 2-D wavelet of shape (nt0, nwav) holds
    one wavelet per time sample, and as pylops builds it ``Cop = MatrixMult(nonstationary_convmtx(wav, nt0,
    hc=nwav // 2, pad=(nt0, nt0)), otherdims=spatdims)`` and the operator is ``Cop * FirstDerivative(dims, axis=0,
    sampling=1.0, kind=kind)``; another first dimension raises pylops' ``ValueError``."""
    wav = np.asarray(wav)
    if wav.ndim != 2:
        return poststack.PoststackLinearModelling(wav, nt0, spatdims=spatdims, explicit=explicit, sparse=sparse,
                                                  kind=kind)
    if wav.shape[0] != nt0:
        raise ValueError("Provide 1d wavelet or 2d wavelet composed of nt0 wavelets")
    if explicit or sparse or np.iscomplexobj(wav):
        raise NotImplementedError("only the matrix-free operator with a real wavelet is restated")
    if kind not in ("forward", "centered"):
        raise NotImplementedError(f"{kind} not an available derivative kind...")
    if spatdims is None:
        dims = (nt0,)
    elif np.ndim(spatdims) == 0:
        dims = (nt0, spatdims)
    else:
        dims = (nt0,) + tuple(spatdims)
    C = nonstationary_convmtx(wav, nt0, hc=wav.shape[1] // 2, pad=(nt0, nt0))
    Cop = MatrixMult(C, otherdims=dims[1:], dtype=wav.dtype)
    Dop = FirstDerivative(dims, axis=0, sampling=1.0, kind=kind, dtype=wav.dtype)
    return ProductLinearOperator(Cop, Dop)             # pylops' Cop * Dop
