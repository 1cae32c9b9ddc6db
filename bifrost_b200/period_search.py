"""bf.period_search.PeriodSearch: whitened, harmonic-summed power spectra of
a dispersion bank's FFTs (extension, bfPeriodSearch*; include/bifrost_b200.h).

For each row of in [..., nbin] cf32 (the r2c spectrum of one DM trial's time
series), each harmonic level l (nharm 2^l) and each `decim` bins: the largest
sum S of the whitened power at the l-th set of harmonics, as
out [..., nlevel, nblk, 2] f32 holding (power, bin offset in the block).
`significance` turns a power of level l into a Gaussian-equivalent sigma, so
peaks of different levels can be ranked against each other."""
import math

import numpy as np

from bifrost_b200.libbifrost import _bf, _check, _exec_storage, BifrostObject
from bifrost_b200.ndarray import asarray

NHARM = (1, 2, 4, 8, 16, 32)


def output_nlevel(nharm):
    """Harmonic levels 1, 2, 4, .., nharm."""
    return int(nharm).bit_length()


def output_nblock(nbin, decim):
    """Number of `decim`-bin blocks in `nbin` bins."""
    return -(-int(nbin) // int(decim))


class PeriodSearch(BifrostObject):
    def __init__(self):
        BifrostObject.__init__(self, _bf.bfPeriodSearchCreate, _bf.bfPeriodSearchDestroy)

    def init(self, nharm, window, decim):
        _check(_bf.bfPeriodSearchInit(self.obj, int(nharm), int(window), int(decim)))
        self.nharm, self.window, self.decim = int(nharm), int(window), int(decim)

    def _run(self, idata, odata, **storage):
        return _exec_storage(_bf.bfPeriodSearchExecute, self.obj, asarray(idata).as_BFarray(),
                             asarray(odata).as_BFarray(), **storage)

    def execute(self, idata, odata):
        self._run(idata, odata)
        return odata

    def get_workspace_size(self, idata, odata):
        return self._run(idata, odata, query=True)

    def execute_workspace(self, idata, odata, workspace_ptr, workspace_size):
        self._run(idata, odata, workspace=(workspace_ptr, workspace_size))
        return odata


# ---- significance -----------------------------------------------------------
_LOG_SQRT_2PI = 0.5 * math.log(2 * math.pi)
_NTERM = 40            # series / continued-fraction terms: 1e-14 at x = 3


def _log_norm_sf(x):
    """(log(1 - Phi(x)), pdf / sf) for x >= 0, to about 1e-14 relative.
    Below 3 the power series of Phi(x) - 1/2; from 3 up the continued
    fraction of the Mills ratio sf / pdf, evaluated backwards."""
    log_pdf = -0.5 * x * x - _LOG_SQRT_2PI
    log_sf = np.empty_like(x)
    small = x < 3.0
    xs = x[small]
    term = xs.copy()
    acc = xs.copy()
    for n in range(1, _NTERM):
        term *= xs * xs / (2 * n + 1)
        acc += term
    log_sf[small] = np.log(0.5 - np.exp(log_pdf[small]) * acc)
    xl = x[~small]
    r = np.zeros_like(xl)
    for n in range(_NTERM, 0, -1):
        r = n / (xl + r)
    log_sf[~small] = log_pdf[~small] - np.log(xl + r)
    return log_sf, np.exp(log_pdf - log_sf)


def _norm_isf_log(log_q):
    """x >= 0 with log(1 - Phi(x)) = log_q, for log_q <= log(1/2).  Newton's
    method on the concave log tail, started at sqrt(-2 log_q), which lies to the
    right of the root (1 - Phi(x) < exp(-x^2 / 2) / 2 there), so it converges
    monotonically from that side."""
    x = np.sqrt(-2.0 * log_q)
    for _ in range(50):
        f, hazard = _log_norm_sf(x)
        step = (f - log_q) / hazard
        x = np.maximum(x + step, 0.0)
        if not np.any(np.abs(step) > 1e-13 * np.maximum(x, 1.0)):
            break
    return x


def _log_gamma_tails(s, h):
    """(log Q, log(1 - Q)) of a sum of h Exp(1) variables at s > 0, with
    Q = exp(-s) sum_{j<h} s^j / j!: the finite sum for Q, and for 1 - Q the
    series exp(-s) s^h / h! sum_n s^n h! / (h + n)! where s < h + 1 (it sums
    terms that decay at least as fast as s / (h + n)), -expm1(log Q) elsewhere."""
    log_s = np.log(s)
    terms = [np.zeros_like(s)] + [j * log_s - math.lgamma(j + 1) for j in range(1, h)]
    top = np.maximum.reduce(terms)
    log_q = np.minimum(-s + top + np.log(sum(np.exp(t - top) for t in terms)), 0.0)
    near = s < h + 1
    sn = s[near]
    term = np.ones_like(sn)
    acc = np.ones_like(sn)
    for n in range(1, 200):
        term *= sn / (h + n)
        acc += term
    log_p = np.empty_like(s)
    log_p[near] = -sn + h * np.log(sn) - math.lgamma(h + 1) + np.log(acc)
    log_p[~near] = np.log(-np.expm1(log_q[~near]))
    return log_q, log_p


def significance(power, nharm):
    """Gaussian-equivalent sigma of a harmonic sum `power` of `nharm` whitened
    noise bins: S, the sum of nharm Exp(1) variables, exceeds `power` with
    probability Q = exp(-S) sum_{j < nharm} S^j / j!, and sigma = Phi^-1(1 - Q).
    Evaluated in log space, so powers up to 1e4 stay finite; power 0 gives
    -inf.  numpy and math only."""
    s = np.asarray(power, np.float64)
    flat = np.maximum(s.ravel(), 0.0)
    sigma = np.full(flat.shape, -np.inf)
    pos = flat > 0
    log_q, log_p = _log_gamma_tails(flat[pos], int(nharm))
    upper = log_q <= log_p              # Q <= 1/2: sigma >= 0
    x = _norm_isf_log(np.where(upper, log_q, log_p))
    sigma[pos] = np.where(upper, x, -x)
    sigma = sigma.reshape(s.shape)
    return sigma if sigma.ndim else float(sigma)
