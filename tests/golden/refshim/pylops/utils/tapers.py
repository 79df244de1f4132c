"""Restatement of third-party ``pylops.utils.tapers`` (pylops 2.x, as remembered: pylops is not installed here to
check it) -- TEST INFRASTRUCTURE for the restated Sliding2D / Sliding3D.  A taper of ``nmask`` samples rises over its
first ``ntap`` samples and falls, mirrored, over its last ``ntap``, with ones between:

- ``"hanning"``: the first ``ntap`` samples of ``np.hanning(2 * ntap - 1)``; ``ValueError`` when ``nmask // ntap < 2``;
- ``"cosine"`` / ``"cosinesquare"``: the first ``ntap`` samples of ``(0.5 * (cos((k - c) * pi / c) + 1)) ** e`` over
  ``k < 2 * ntap - 1`` with ``c = ntap - 1``, ``e`` 1 or 2 (``ntap = 1`` is taken as 0);
- anything else (``None``): ones.

``taper2d`` tiles the taper along a second axis of ``nt`` samples, ``taper3d`` is the outer product of two tapers
tiled along a third."""
import numpy as np


def hanningtaper(nmask, ntap):
    if ntap > 0 and (nmask // ntap) < 2:
        ntap_min = nmask / 2 if nmask % 2 == 0 else (nmask - 1) / 2
        raise ValueError(f"ntap={ntap} must be smaller or equal than {ntap_min}")
    han_win = np.hanning(ntap * 2 - 1)
    st_tpr = han_win[:ntap]
    return np.concatenate([st_tpr, np.ones(nmask - 2 * ntap), np.flipud(st_tpr)])


def cosinetaper(nmask, ntap, square=False):
    ntap = 0 if ntap == 1 else ntap
    exponent = 2 if square else 1
    c = (ntap * 2 - 2) / 2
    with np.errstate(divide="ignore", invalid="ignore"):
        cos_win = (0.5 * (np.cos((np.arange(ntap * 2 - 1) - c) * np.pi / c) + 1.0)) ** exponent
    st_tpr = cos_win[:ntap]
    return np.concatenate([st_tpr, np.ones(nmask - 2 * ntap), np.flipud(st_tpr)])


def taper(nmask, ntap, tapertype):
    if tapertype == "hanning":
        return hanningtaper(nmask, ntap)
    if tapertype == "cosine":
        return cosinetaper(nmask, ntap, False)
    if tapertype == "cosinesquare":
        return cosinetaper(nmask, ntap, True)
    return np.ones(nmask)


def taper2d(nt, nmask, ntap, tapertype="hanning"):
    return np.tile(taper(nmask, ntap, tapertype)[:, np.newaxis], (1, nt))


def taper3d(nt, nmask, ntap, tapertype="hanning"):
    tpr_y = taper(nmask[0], ntap[0], tapertype)
    tpr_x = taper(nmask[1], ntap[1], tapertype)
    return np.tile(np.outer(tpr_y, tpr_x)[:, :, np.newaxis], (1, 1, nt))
