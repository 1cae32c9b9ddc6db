"""bf.fold.Fold: phase-binned pulsar profiles of a topocentric spin model
(extension, bfFold*; include/bifrost_b200.h).

Each row of x [nchan, ..., ntime] (u8, u16 or f32) is folded into `nbin`
phase bins: out [nchan, ..., nbin] f32 gets the per-bin sums and count
[nchan, nbin] i32 the samples of each channel per bin.  Sample t of channel c
is at tau = t0 - delay[c] + (first + t) tsamp seconds from the ephemeris
epoch and has phase ((nuddot/6 tau + nudot/2) tau + nu) tau turns."""
import ctypes

import numpy as np

from bifrost_b200.libbifrost import _bf, _check, _exec_storage, BifrostObject
from bifrost_b200.ndarray import asarray
from bifrost_b200.coherent_dedisp import KDM

NBIN_MAX = 4096


def dispersion_delays(freqs_mhz, dm, fref_mhz):
    """Cold-plasma delays in seconds of frequencies `freqs_mhz` relative to
    `fref_mhz`: KDM dm (f^-2 - fref^-2), fp64 [len(freqs)]."""
    f = np.asarray(freqs_mhz, dtype=np.float64)
    return KDM * float(dm) * (f ** -2 - float(fref_mhz) ** -2)


class Fold(BifrostObject):
    def __init__(self):
        BifrostObject.__init__(self, _bf.bfFoldCreate, _bf.bfFoldDestroy)

    def init(self, nbin, delays, tsamp, t0, nu, nudot=0.0, nuddot=0.0):
        """nbin phase bins (1 ... 4096), per-channel delays in s (fp64, one per
        channel), sample interval tsamp s, t0 = the time of stream sample 0 at
        the reference frequency in s from the ephemeris epoch, spin frequency
        nu Hz and its derivatives nudot Hz/s, nuddot Hz/s^2."""
        d = np.ascontiguousarray(np.asarray(delays, dtype=np.float64).reshape(-1))
        _check(_bf.bfFoldInit(self.obj, int(nbin), d.size, d.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                              float(tsamp), float(t0), float(nu), float(nudot), float(nuddot)))
        self.nbin, self.nchan = int(nbin), int(d.size)
        self.delays = d
        self.tsamp, self.t0 = float(tsamp), float(t0)
        self.nu, self.nudot, self.nuddot = float(nu), float(nudot), float(nuddot)

    def _run(self, idata, odata, count, first, accumulate, **storage):
        return _exec_storage(_bf.bfFoldExecute, self.obj, asarray(idata).as_BFarray(), int(first),
                             asarray(odata).as_BFarray(), asarray(count).as_BFarray(), int(bool(accumulate)),
                             **storage)

    def execute(self, idata, odata, count, first=0, accumulate=False):
        """Fold idata, whose sample 0 is stream sample `first`, into odata (f32
        sums) and count (i32): overwrite them, or add to them with
        accumulate=True."""
        self._run(idata, odata, count, first, accumulate)
        return odata

    def get_workspace_size(self, idata, odata, count):
        return self._run(idata, odata, count, 0, False, query=True)

    def execute_workspace(self, idata, odata, count, workspace_ptr, workspace_size, first=0, accumulate=False):
        self._run(idata, odata, count, first, accumulate, workspace=(workspace_ptr, workspace_size))
        return odata
