"""Periodicity-search oracle (numpy, fp64).  TEST INFRASTRUCTURE -- see
oracle/__init__.py.

The semantics of bfPeriodSearchExecute (include/bifrost_b200.h), restated with
the same fp64 operation order (numpy rounds every operation once and never
contracts, so it gives the library's bits):
  P[k] = re re + im im, re and im widened from f32;
  med_j = the element of rank (m_j - 1) // 2 of window j's P (np.partition);
  p[0] = 0, p[k] = float32((P[k] / med_j) * LN2) if med_j > 0 else 0;
  S_1 = p, S_h = S_{h/2} + T_h, T_h[k] = sum over odd i < h ascending of
  p[(2 i k + h) // (2 h)];
  block j of level l: the first argmax k of S_h over [j decim, (j+1) decim),
  reported as (float32(S_h[k]), k - j decim).
"""
import numpy as np

LN2 = 0.6931471805599453


def whiten(spec, window):
    """p [..., nbin] f32 of a cf32 spectrum [..., nbin]."""
    spec = np.asarray(spec, np.complex64)
    re = spec.real.astype(np.float64)
    im = spec.imag.astype(np.float64)
    P = re * re + im * im
    nbin = P.shape[-1]
    p = np.zeros(P.shape, np.float32)
    for k0 in range(0, nbin, window):
        w = P[..., k0:k0 + window]
        r = (w.shape[-1] - 1) // 2
        med = np.partition(w, r, axis=-1)[..., r:r + 1]
        with np.errstate(divide='ignore', invalid='ignore'):
            q = ((w / med) * LN2).astype(np.float32)
        p[..., k0:k0 + window] = np.where(med > 0, q, np.float32(0))
    p[..., 0] = 0
    return p


def harmonic_sums(p, nharm):
    """[S_1, S_2, .., S_nharm] fp64, each [..., nbin], from p [..., nbin] f32."""
    p64 = np.asarray(p, np.float32).astype(np.float64)
    k = np.arange(p64.shape[-1], dtype=np.int64)
    S = [p64]
    h = 2
    while h <= nharm:
        t = np.zeros_like(p64)
        for i in range(1, h, 2):
            t = t + p64[..., (2 * i * k + h) // (2 * h)]
        S.append(S[-1] + t)
        h *= 2
    return S


def peaks(S, decim):
    """out [..., nlevel, nblk, 2] f32 from the level sums."""
    nbin = S[0].shape[-1]
    nblk = -(-nbin // decim)
    lead = S[0].shape[:-1]
    out = np.zeros(lead + (len(S), nblk, 2), np.float32)
    pad = nblk * decim - nbin
    for l, s in enumerate(S):
        sp = np.concatenate([s, np.full(lead + (pad,), -np.inf)], axis=-1)
        sp = sp.reshape(lead + (nblk, decim))
        with np.errstate(invalid='ignore'):
            kb = np.argmax(sp, axis=-1)                 # first maximum
        out[..., l, :, 0] = np.take_along_axis(sp, kb[..., None], axis=-1)[..., 0].astype(np.float32)
        out[..., l, :, 1] = kb.astype(np.float32)
    return out


def period_search(spec, nharm, window, decim):
    """out [..., nlevel, nblk, 2] f32 of a cf32 spectrum [..., nbin]."""
    return peaks(harmonic_sums(whiten(spec, window), nharm), decim)
