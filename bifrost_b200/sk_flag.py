"""bf.sk_flag.SkFlag: RFI excision by windowed spectral kurtosis (extension,
bfSkFlag*; include/bifrost_b200.h).

For each row of x [..., ntime] (u8, u16 or f32 power) and each window of
`window` samples, the spectral kurtosis estimator sk; windows outside
[lo, hi] are replaced by the mean of the row's clean samples.  y has x's
dtype and shape and may be x itself."""
import math

from bifrost_b200.libbifrost import _bf, _check, _exec_storage, BifrostObject
from bifrost_b200.ndarray import asarray


def sk_variance(window, nacc=1, shape=1.0):
    """Var[sk] for Gamma(nacc * shape)-distributed power in windows of m =
    `window` samples (Nita & Gary 2010): 2 m^2 Nd (Nd + 1) /
    ((m - 1)(m Nd + 2)(m Nd + 3)) with Nd = nacc * shape.  E[sk] = 1."""
    m, nd = float(window), float(nacc) * float(shape)
    return 2 * m * m * nd * (nd + 1) / ((m - 1) * (m * nd + 2) * (m * nd + 3))


def sk_thresholds(window, nacc=1, shape=1.0, sigma=3.0):
    """(lo, hi) = 1 -/+ sigma * sqrt(Var[sk]).

    The distribution of sk is skewed (a long upper tail) for small windows,
    so these symmetric bounds flag about 1 % of clean windows at sigma = 3,
    not the 0.27 % of a normal distribution."""
    s = float(sigma) * math.sqrt(sk_variance(window, nacc, shape))
    return 1.0 - s, 1.0 + s


def sk_nwindow(ntime, window):
    """Number of windows (the last may be short) in `ntime` samples."""
    return -(-int(ntime) // int(window))


def _arr(a):
    return None if a is None else asarray(a).as_BFarray()


class SkFlag(BifrostObject):
    def __init__(self):
        BifrostObject.__init__(self, _bf.bfSkFlagCreate, _bf.bfSkFlagDestroy)

    def init(self, window, nacc=1, shape=1.0, lo=None, hi=None):
        """lo and hi default to sk_thresholds(window, nacc, shape) (3 sigma)."""
        if lo is None and hi is None:
            lo, hi = sk_thresholds(window, nacc, shape)
        elif lo is None or hi is None:
            raise ValueError("give both thresholds or neither")
        _check(_bf.bfSkFlagInit(self.obj, int(window), int(nacc), float(shape), float(lo), float(hi)))
        self.window, self.nacc, self.shape = int(window), int(nacc), float(shape)
        self.lo, self.hi = float(lo), float(hi)

    def _run(self, idata, odata, sk, **storage):
        return _exec_storage(_bf.bfSkFlagExecute, self.obj, asarray(idata).as_BFarray(),
                             asarray(odata).as_BFarray(), _arr(sk), **storage)

    def execute(self, idata, odata, sk=None):
        """y = odata (may be idata) from x = idata; sk, if given, receives the
        f32 [..., nwin] statistic."""
        self._run(idata, odata, sk)
        return odata

    def get_workspace_size(self, idata, odata, sk=None):
        return self._run(idata, odata, sk, query=True)

    def execute_workspace(self, idata, odata, workspace_ptr, workspace_size, sk=None):
        self._run(idata, odata, sk, workspace=(workspace_ptr, workspace_size))
        return odata
