"""bf.pulse_search.PulseSearch: boxcar matched-filter search of a dispersion
bank (extension, bfPulseSearch*; include/bifrost_b200.h).

For each row of x [..., ndm, ntime] f32 and each `decim` starts, the peak
S/N over the boxcar widths: out [..., ndm, nblk, 3] f32 holding
(snr, start offset in the block, width)."""
import ctypes

from bifrost_b200.libbifrost import _bf, _check, _exec_storage, BifrostObject
from bifrost_b200.ndarray import asarray


def output_nblock(ntime, widths, decim):
    """Number of `decim`-start blocks searched in `ntime` samples."""
    nout = int(ntime) - max(widths) + 1
    return -(-nout // int(decim)) if nout > 0 else 0


class PulseSearch(BifrostObject):
    def __init__(self):
        BifrostObject.__init__(self, _bf.bfPulseSearchCreate, _bf.bfPulseSearchDestroy)

    def init(self, widths, decim):
        widths = [int(w) for w in widths]
        arr = (ctypes.c_int * max(1, len(widths)))(*widths)
        _check(_bf.bfPulseSearchInit(self.obj, len(widths), arr, int(decim)))
        self.widths, self.decim = widths, int(decim)

    def _run(self, idata, odata, **storage):
        return _exec_storage(_bf.bfPulseSearchExecute, self.obj, asarray(idata).as_BFarray(),
                             asarray(odata).as_BFarray(), **storage)

    def execute(self, idata, odata):
        self._run(idata, odata)
        return odata

    def get_workspace_size(self, idata, odata):
        return self._run(idata, odata, query=True)

    def execute_workspace(self, idata, odata, workspace_ptr, workspace_size):
        self._run(idata, odata, workspace=(workspace_ptr, workspace_size))
        return odata
