"""bf.coherent_dedisp.CoherentDedisp: coherent dedispersion of critically
sampled complex baseband channels (extension, bfCoherentDedisp*;
include/bifrost_b200.h).

Each channel of x [nchan, ..., ntime] (ci4, ci8, ci16 or cf32 voltages) is
filtered by overlap-save with N-point segments and the inverse of the
cold-plasma transfer function, which aligns every output sample to the
arrival time at its channel's top edge.  Output t depends on the input from
t to t + overlap.  The output is cf32; integer inputs enter unscaled.

CoherentDedisp.filterbank does the same filtering, splits each channel into
nfine fine channels, detects and sums nint samples in one pass, and writes
only f32 power (bfCoherentDedispFilterbank)."""
import math

from bifrost_b200.libbifrost import _bf, _check, _exec_storage, _get, BifrostObject
from bifrost_b200.map import DETECT_MODES
from bifrost_b200.ndarray import asarray

KDM = 4.148741601e3          # MHz^2 pc^-1 cm^3 s
NFFT_MIN, NFFT_MAX = 256, 1 << 20


def dispersion_overlap(nchan, f0, df, dm):
    """M: the dispersion smear of the worst channel in samples,
    ceil(max_c D DM ((f_c - |df|/2)^-2 - (f_c + |df|/2)^-2) |df| 1e6) with
    f_c = f0 + c df MHz.  0 at DM 0."""
    adf = abs(float(df))
    smear = 0.0
    for c in range(int(nchan)):
        fc = float(f0) + c * float(df)
        lo, top = fc - 0.5 * adf, fc + 0.5 * adf
        if lo <= 0:
            raise ValueError("channel %d has its bottom edge at %g MHz" % (c, lo))
        smear = max(smear, KDM * float(dm) * (1.0 / (lo * lo) - 1.0 / (top * top)) * adf * 1e6)
    return int(math.ceil(smear))


def default_nfft(overlap):
    """The smallest power of two >= max(256, 4 overlap), which keeps at least
    three quarters of every segment; ValueError above 2^20."""
    n = NFFT_MIN
    while n < 4 * int(overlap):
        n *= 2
    if n > NFFT_MAX:
        raise ValueError("an overlap of %d samples needs nfft %d > 2^20" % (overlap, n))
    return n


def filterbank_shape(nchan, nb, ntime, nfine=1, mode='scalar', nint=1):
    """The f32 output shape of CoherentDedisp.filterbank on [nchan, nb, ntime]:
    [nchan nfine, P, ntime / (nfine nint)] with P = nb for 'scalar', else the
    products of the mode (4 stokes / coherence, 1 stokes_i).  ValueError when
    ntime is not a multiple of nfine nint."""
    nchan, nb, ntime, nfine, nint = int(nchan), int(nb), int(ntime), int(nfine), int(nint)
    if mode not in ('scalar', 'stokes', 'stokes_i', 'coherence'):
        raise ValueError("mode must be 'scalar', 'stokes', 'stokes_i' or 'coherence', got %r" % (mode,))
    if nfine < 1 or nint < 1 or ntime % (nfine * nint):
        raise ValueError("ntime (%d) must be a multiple of nfine (%d) x nint (%d)" % (ntime, nfine, nint))
    nprod = nb if mode == 'scalar' else 1 if mode == 'stokes_i' else 4
    return (nchan * nfine, nprod, ntime // (nfine * nint))


def _mode(mode):
    return DETECT_MODES[mode] if isinstance(mode, str) else int(mode)


class CoherentDedisp(BifrostObject):
    def __init__(self):
        BifrostObject.__init__(self, _bf.bfCoherentDedispCreate, _bf.bfCoherentDedispDestroy)

    def init(self, nchan, f0, df, dm, nfft):
        """Channels f0 + c df MHz (c < nchan), dispersion measure dm in
        pc cm^-3, nfft-point segments."""
        _check(_bf.bfCoherentDedispInit(self.obj, int(nchan), float(f0), float(df), float(dm), int(nfft)))
        self.nchan, self.f0, self.df, self.dm, self.nfft = int(nchan), float(f0), float(df), float(dm), int(nfft)
        self.overlap = int(_get(_bf.bfCoherentDedispGetOverlap, self.obj))

    def _run(self, idata, odata, **storage):
        return _exec_storage(_bf.bfCoherentDedispExecute, self.obj, asarray(idata).as_BFarray(),
                             asarray(odata).as_BFarray(), **storage)

    def execute(self, idata, odata):
        """odata (cf32, idata's shape) = idata dedispersed."""
        self._run(idata, odata)
        return odata

    def get_workspace_size(self, idata, odata):
        return self._run(idata, odata, query=True)

    def execute_workspace(self, idata, odata, workspace_ptr, workspace_size):
        self._run(idata, odata, workspace=(workspace_ptr, workspace_size))
        return odata

    def _run_filterbank(self, idata, odata, nfine, mode, nint, **storage):
        return _exec_storage(_bf.bfCoherentDedispFilterbank, self.obj, asarray(idata).as_BFarray(), int(nfine),
                             _mode(mode), int(nint), asarray(odata).as_BFarray(), **storage)

    def filterbank(self, idata, odata, nfine=1, mode='scalar', nint=1):
        """odata (f32 filterbank_shape(...)) = idata [nchan, nb, ntime]
        dedispersed, split into nfine fine channels per channel, detected with
        `mode` ('scalar', 'stokes', 'stokes_i', 'coherence'; polarised modes
        take rows 0, 1 as x, y) and summed over nint fine samples.  With
        nfine = 1 and nint dividing N - M: detect(execute(idata), mode)
        reduced over nint, bit for bit."""
        self._run_filterbank(idata, odata, nfine, mode, nint)
        return odata

    def get_filterbank_workspace_size(self, idata, odata, nfine=1, mode='scalar', nint=1):
        return self._run_filterbank(idata, odata, nfine, mode, nint, query=True)

    def filterbank_workspace(self, idata, odata, workspace_ptr, workspace_size, nfine=1, mode='scalar', nint=1):
        self._run_filterbank(idata, odata, nfine, mode, nint, workspace=(workspace_ptr, workspace_size))
        return odata
