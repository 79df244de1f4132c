"""Restatement of third-party ``pylops.waveeqprocessing.LSM`` (pylops 2.x, kind="kirchhoff") -- TEST INFRASTRUCTURE
for tests/golden/make_golden_kirchhoff.py: only the demigration operator ``Demop`` that tutorials/lsm.py uses."""
from .kirchhoff import Kirchhoff


class LSM:
    def __init__(self, z, x, t, srcs, recs, vel, wav, wavcenter, y=None, kind="kirchhoff", dottest=False,
                 **kwargs_mod):
        if kind != "kirchhoff" or dottest:
            raise NotImplementedError("only kind='kirchhoff' without dottest is restated")
        self.y, self.x, self.z, self.t = y, x, z, t
        self.Demop = Kirchhoff(z, x, t, srcs, recs, vel, wav, wavcenter, y=y, **kwargs_mod)
