"""Pulsar folding oracle (numpy, fp64).  TEST INFRASTRUCTURE -- see
oracle/__init__.py.

The semantics of bfFoldExecute (include/bifrost_b200.h), restated with the
same fp64 operation order (numpy rounds every operation once and never
contracts, so every bin is the library's):
  a_c  = t0 - delay[c]
  tau  = a_c + (double)(first + t) * tsamp
  phi  = ((c3 tau + c2) tau + nu) tau      c2 = 0.5 nudot, c3 = nuddot / 6.0
  frac = phi - floor(phi)
  bin  = min((int)floor(frac * nbin), nbin - 1)
out[row][bin] = fp64 sum of the row's samples in the bin; count[c][bin] = the
number of channel c's samples in it.
"""
import numpy as np


def bins(nchan, ntime, nbin, delays, tsamp, t0, nu, nudot=0.0, nuddot=0.0, first=0):
    """int64 [nchan, ntime]: the bin of every sample."""
    a = (np.float64(t0) - np.asarray(delays, np.float64)).reshape(nchan, 1)
    t = (np.int64(first) + np.arange(ntime, dtype=np.int64)).astype(np.float64)
    tau = a + t * np.float64(tsamp)
    c2 = np.float64(0.5) * np.float64(nudot)
    c3 = np.float64(nuddot) / np.float64(6.0)
    phi = ((c3 * tau + c2) * tau + np.float64(nu)) * tau
    frac = phi - np.floor(phi)
    return np.minimum(np.floor(frac * np.float64(nbin)).astype(np.int64), nbin - 1)


def fold(x, nbin, delays, tsamp, t0, nu, nudot=0.0, nuddot=0.0, first=0):
    """(sums fp64 [nchan, ..., nbin], counts int64 [nchan, nbin]) of x
    [nchan, ..., ntime] (u8, u16 or f32)."""
    x = np.asarray(x)
    nchan, ntime = x.shape[0], x.shape[-1]
    b = bins(nchan, ntime, nbin, delays, tsamp, t0, nu, nudot, nuddot, first)
    sums = np.zeros(x.shape[:-1] + (nbin,), np.float64)
    counts = np.zeros((nchan, nbin), np.int64)
    for c in range(nchan):
        counts[c] = np.bincount(b[c], minlength=nbin)
        for r in np.ndindex(*x.shape[1:-1]):
            sums[(c,) + r] = np.bincount(b[c], weights=x[(c,) + r].astype(np.float64), minlength=nbin)
    return sums, counts


def fold_nonfinite(x, nbin, delays, tsamp, t0, nu, nudot=0.0, nuddot=0.0, first=0):
    """fold() for rows that may hold NaN / inf: np.bincount skips nothing but
    adds in its own order, so bins holding both +inf and -inf, or any NaN, are
    NaN here as they are in any order."""
    x = np.asarray(x)
    nchan, ntime = x.shape[0], x.shape[-1]
    b = bins(nchan, ntime, nbin, delays, tsamp, t0, nu, nudot, nuddot, first)
    sums, counts = fold(np.where(np.isfinite(x), x, 0).astype(x.dtype), nbin, delays, tsamp, t0, nu,
                        nudot, nuddot, first)
    for c in range(nchan):
        for r in np.ndindex(*x.shape[1:-1]):
            row = x[(c,) + r].astype(np.float64)
            for k in np.flatnonzero(~np.isfinite(row)):
                sums[(c,) + r + (b[c, k],)] += row[k]
    return sums, counts
