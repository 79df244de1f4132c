"""The lossless integer codec of the exact operator fixtures, and the row split their multi-rank cases use.

A fixture stores an exactly representable output y as the integer ENC * y (ENC a power of two chosen per family, the
integer type the narrowest that holds every value), and the forward / adjoint pair of one case as ``{key}/y`` and
``{key}/ya``, with the imaginary parts of a complex128 case as ``{key}/yi`` and ``{key}/yai``."""
import numpy as np


def rows_of(P, n):
    """rows of an axis of length n per rank (the reference's SCATTER split)"""
    return [n // P + (1 if r < n % P else 0) for r in range(P)]


def encode(y, enc, itype):
    """enc * y as ``itype``, asserting that the value is exact and fits"""
    e = np.rint(np.asarray(y, dtype=np.float64) * enc)
    assert np.array_equal(e / enc, y) and np.abs(e).max() <= np.iinfo(itype).max
    return e.astype(itype)


def decode(gold, key, dt, enc):
    """the (forward, adjoint) outputs stored under ``key``, decoded in dtype dt (enc 1: stored as float64)"""
    f = [gold[f"{key}/{n}"].astype(np.float64) / enc for n in ("y", "ya", "yi", "yai")[:4 if dt == "complex128" else 2]]
    if dt == "complex128":
        return f[0] + 1j * f[2], f[1] + 1j * f[3]
    return f[0].astype(dt), f[1].astype(dt)
