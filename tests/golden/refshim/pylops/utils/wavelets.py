"""Restatement of third-party ``pylops.utils.wavelets.ricker`` (pylops 2.x) -- TEST INFRASTRUCTURE for
tests/golden/make_golden_kirchhoff.py (tutorials/lsm.py builds its wavelet with it)."""
import numpy as np


def ricker(t, f0=10, taper=None):
    """Ricker wavelet on the symmetric time axis built from the one-sided ``t`` (an even-length ``t`` loses its last
    sample); returns the wavelet, its time axis and the index of its peak ``wcenter``"""
    if len(t) % 2 == 0:
        t = t[:-1]
    w = (1 - 2 * (np.pi * f0 * t) ** 2) * np.exp(-((np.pi * f0 * t) ** 2))
    w = np.concatenate((np.flipud(w[1:]), w), axis=0)
    t = np.concatenate((np.flipud(-t[1:]), t), axis=0)
    if taper is not None:
        w = w * taper(len(t))
    wcenter = np.argmax(np.abs(w))
    return w, t, wcenter
