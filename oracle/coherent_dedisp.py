"""Coherent dedispersion oracle (numpy, fp64).  TEST INFRASTRUCTURE -- see
oracle/__init__.py.

The definition of bfCoherentDedispExecute (include/bifrost_b200.h):
  channel c: f_c = f0 + c df MHz, f_top = f_c + |df|/2, sample 1/|df| us;
  M = ceil(max_c D DM ((f_c - |df|/2)^-2 - f_top^-2) |df| 1e6);
  nu_k = fftfreq(N)[k] df, K = D DM 1e6,
  phi_k = sgn(df) K [nu_k (f_c^-2 - f_top^-2) - nu_k^2 / (f_c^2 (f_c + nu_k))],
  H_k = exp(2 pi i phi_k);
  segments at s = 0, L, 2L, .. (L = N - M) while s < ntime, N samples each
  (zeros past the end), y = IFFT(H FFT(x_seg)) / N, out[s : s + L] = y[:L].
conj(H) is the dispersion itself (disperse), with group delay
D DM (f^-2 - f_top^-2) at sky frequency f = f_c + nu.
"""
import numpy as np

KDM = 4.148741601e3          # MHz^2 pc^-1 cm^3 s


def overlap(nchan, f0, df, dm):
    """M, the smear of the worst channel in samples."""
    adf = abs(float(df))
    fc = float(f0) + np.arange(int(nchan), dtype=np.float64) * float(df)
    lo, top = fc - 0.5 * adf, fc + 0.5 * adf
    smear = KDM * float(dm) * (1.0 / (lo * lo) - 1.0 / (top * top)) * adf * 1e6
    return int(np.ceil(smear.max())) if len(smear) else 0


def phase(n, fc, df, dm):
    """phi_k in cycles, fp64 [n], for a channel centred on fc MHz."""
    df = float(df)
    nu = np.fft.fftfreq(int(n)) * df
    top = fc + 0.5 * abs(df)
    phi = KDM * float(dm) * 1e6 * (nu * (1.0 / (fc * fc) - 1.0 / (top * top)) - nu * nu / (fc * fc * (fc + nu)))
    return np.sign(df) * phi


def chirp(n, fc, df, dm):
    """H_k = exp(2 pi i phi_k), complex128 [n], phi reduced modulo one turn first."""
    phi = phase(n, fc, df, dm)
    phi = phi - np.rint(phi)
    return np.exp(2j * np.pi * phi)


def _as_complex(x):
    x = np.asarray(x)
    if np.iscomplexobj(x):
        return x.astype(np.complex128)
    return x['re'].astype(np.float64) + 1j * x['im'].astype(np.float64)


def dedisperse(x, f0, df, dm, nfft):
    """The segmented operation on x [nchan, ..., ntime] (complex, or a
    structured re/im integer array): complex128 of x's shape."""
    x = _as_complex(x)
    nchan, ntime = x.shape[0], x.shape[-1]
    m = overlap(nchan, f0, df, dm)
    step = nfft - m
    if step <= 0:
        raise ValueError("overlap %d >= nfft %d" % (m, nfft))
    out = np.zeros(x.shape, np.complex128)
    nseg = -(-ntime // step)
    pad = np.zeros(x.shape[:-1] + (nseg * step + nfft - ntime,), np.complex128)
    xp = np.concatenate([x, pad], axis=-1)
    for c in range(nchan):
        h = chirp(nfft, float(f0) + c * float(df), df, dm)
        segs = np.stack([xp[c, ..., s * step:s * step + nfft] for s in range(nseg)], axis=-2)
        y = np.fft.ifft(np.fft.fft(segs, axis=-1) * h, axis=-1)[..., :step]
        out[c] = y.reshape(y.shape[:-2] + (nseg * step,))[..., :ntime]
    return out


def disperse(x, f0, df, dm):
    """conj(H) over one FFT of the whole row: the dispersion that dedisperse
    undoes (circular: test data should leave M samples of margin)."""
    x = _as_complex(x)
    nchan, n = x.shape[0], x.shape[-1]
    out = np.empty(x.shape, np.complex128)
    for c in range(nchan):
        h = chirp(n, float(f0) + c * float(df), df, dm)
        out[c] = np.fft.ifft(np.fft.fft(x[c], axis=-1) * np.conj(h), axis=-1)
    return out
