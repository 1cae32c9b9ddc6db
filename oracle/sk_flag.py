"""Spectral-kurtosis RFI excision oracle (numpy, fp64).  TEST INFRASTRUCTURE
-- see oracle/__init__.py.

The semantics of bfSkFlagExecute (include/bifrost_b200.h), restated with the
same fp64 operation order (numpy rounds every operation once and never
contracts, so integer inputs give the library's bits):
  window j of a row = samples [j M, min((j+1) M, ntime)), m samples;
  S1 = sum x, S2 = sum x^2: exact uint64 sums for u8 / u16, fp64 for f32;
  a = ((m N) d + 1) / (m - 1); sk = a ((m S2) / (S1 S1) - 1);
  flagged = not (lo <= sk <= hi);
  fill = (sum of S1 over clean windows, ascending) / (their sample count),
  0 if every window is flagged, rounded to nearest even into the dtype;
  y = x on clean windows, fill on flagged ones.
"""
import numpy as np


def window_sums(x, window):
    """(S1, S2, m) per window, fp64 [..., nwin] (m: int64 [nwin])."""
    x = np.asarray(x)
    ntime = x.shape[-1]
    nwin = -(-ntime // window)
    pad = nwin * window - ntime
    if x.dtype in (np.uint8, np.uint16):
        w = x.astype(np.uint64)
        w = np.concatenate([w, np.zeros(x.shape[:-1] + (pad,), np.uint64)], axis=-1)
        w = w.reshape(x.shape[:-1] + (nwin, window))
        s1 = w.sum(axis=-1, dtype=np.uint64).astype(np.float64)
        s2 = (w * w).sum(axis=-1, dtype=np.uint64).astype(np.float64)
    elif x.dtype == np.float32:
        w = x.astype(np.float64)
        w = np.concatenate([w, np.zeros(x.shape[:-1] + (pad,), np.float64)], axis=-1)
        w = w.reshape(x.shape[:-1] + (nwin, window))
        s1 = w.sum(axis=-1)
        s2 = (w * w).sum(axis=-1)
    else:
        raise TypeError("sk_flag takes u8, u16 or f32 power, got %s" % x.dtype)
    m = np.full(nwin, window, np.int64)
    if nwin:
        m[-1] = ntime - (nwin - 1) * window
    return s1, s2, m


def sk(s1, s2, m, nacc, shape):
    """fp64 sk from the window sums, in the library's operation order."""
    md = m.astype(np.float64)
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        a = ((md * float(nacc)) * float(shape) + 1.0) / (md - 1.0)
        return a * ((md * s2) / (s1 * s1) - 1.0)


def sk_flag(x, window, nacc, shape, lo, hi):
    """(y, sk32, flags, sk64, fill) for x [..., ntime] u8 / u16 / f32."""
    x = np.asarray(x)
    s1, s2, m = window_sums(x, window)
    k = sk(s1, s2, m, nacc, shape)
    flags = ~((lo <= k) & (k <= hi))
    clean = np.where(flags, 0.0, s1)
    total = np.cumsum(clean, axis=-1)[..., -1] if clean.shape[-1] else np.zeros(clean.shape[:-1])
    count = np.where(flags, 0, m).sum(axis=-1)
    with np.errstate(divide='ignore', invalid='ignore'):
        fill = np.where(count > 0, total / np.maximum(count, 1).astype(np.float64), 0.0)
    if x.dtype == np.float32:
        fillx = fill.astype(np.float32)
    else:
        fillx = np.rint(fill).astype(x.dtype)
    per_sample = np.repeat(flags, window, axis=-1)[..., :x.shape[-1]]
    y = np.where(per_sample, fillx[..., None], x).astype(x.dtype)
    return y, k.astype(np.float32), flags, k, fill
