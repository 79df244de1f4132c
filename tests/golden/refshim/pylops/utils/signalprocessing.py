"""Restatement of third-party ``pylops.utils.signalprocessing.nonstationary_convmtx`` (pylops 2.x, as remembered) --
TEST INFRASTRUCTURE for the 2-D wavelet branch of refshim's ``pylops.avo.poststack``."""
import numpy as np


def nonstationary_convmtx(H, n, hc=0, pad=(0, 0)):
    """dense (n, n) matrix whose column ``j`` is filter ``H[j]`` centred (``hc``) on row ``j``:
    ``C[i, j] = H[j, hc + i - j]``.  Each padded filter is rolled by its index, then the rows are cut to n."""
    H = np.pad(H, ((0, 0), pad), mode="constant")
    C = np.array([np.roll(h, ih) for ih, h in enumerate(H)])
    C = C[:, pad[0] + hc:pad[0] + hc + n].T
    return C
