"""Coherent filterbank oracle (numpy, fp64).  TEST INFRASTRUCTURE -- see
oracle/__init__.py.

The definition of bfCoherentDedispFilterbank (include/bifrost_b200.h), on top
of the coherent dedispersion of oracle/coherent_dedisp.py: with Nf = N / nfine,
fine channel j of a segment takes bins k = (N/2 + j Nf + q) mod N (q < Nf) of
Y = H_j FFT_N(x_seg) / N, where H_j is the chirp with the fine channel's own
top edge f_top,j = f_c - df/2 + (j + 1/2) df' + |df'|/2 (df' = df / nfine), and
z_j[m] = sum_q Y[k(q)] exp(+2 pi i q m / Nf).  Segments step by
S = q floor((N - M) / q), q = nfine nint, and keep z_j[0 : S / nfine].
Detection as bfDetect, then sums of nint samples.
"""
import numpy as np

from oracle.coherent_dedisp import KDM, overlap, _as_complex


def fine_top(fc, df, nfine, j):
    """Top edge (MHz) of fine channel j of the channel centred on fc."""
    dff = float(df) / nfine
    return fc - 0.5 * float(df) + (j + 0.5) * dff + 0.5 * abs(dff)


def fine_chirp(n, fc, df, dm, nfine):
    """H_k with each bin's fine-channel top edge, complex128 [n], phi reduced
    modulo one turn first."""
    df = float(df)
    nu = np.fft.fftfreq(int(n)) * df
    j = ((np.arange(n) + n // 2) % n) // (n // nfine)
    top = fine_top(fc, df, nfine, j)
    phi = np.sign(df) * KDM * float(dm) * 1e6 * (nu * (1.0 / (fc * fc) - 1.0 / (top * top))
                                                  - nu * nu / (fc * fc * (fc + nu)))
    phi = phi - np.rint(phi)
    return np.exp(2j * np.pi * phi)


def fine_channels(x, f0, df, dm, nfft, nfine, nint=1):
    """z: complex128 [nchan, nfine, nb, ntime / nfine], the fine-channel
    voltages of x [nchan, nb, ntime] with the segment step of nfine nint."""
    x = _as_complex(x)
    nchan, nb, ntime = x.shape
    m = overlap(nchan, f0, df, dm)
    q = nfine * nint
    step = q * ((nfft - m) // q)
    if step <= 0:
        raise ValueError("nfine nint %d > nfft - overlap %d" % (q, nfft - m))
    nf = nfft // nfine
    nseg = -(-ntime // step)
    xp = np.concatenate([x, np.zeros((nchan, nb, nseg * step + nfft - ntime), np.complex128)], axis=-1)
    z = np.zeros((nchan, nfine, nb, ntime // nfine), np.complex128)
    keep = step // nfine
    for c in range(nchan):
        h = fine_chirp(nfft, float(f0) + c * float(df), df, dm, nfine)
        segs = np.stack([xp[c, :, s * step:s * step + nfft] for s in range(nseg)], axis=-2)
        Y = np.fft.fft(segs, axis=-1) * h / nfft
        for j in range(nfine):
            k = (nfft // 2 + j * nf + np.arange(nf)) % nfft
            zj = np.fft.ifft(Y[..., k], axis=-1)[..., :keep] * nf
            z[c, j] = zj.reshape(nb, nseg * keep)[:, :ntime // nfine]
    return z


def detect(z, mode):
    """[..., nb, t] complex -> the products of bfDetect: scalar |z|^2 per row;
    stokes (I, Q, U, V), stokes_i (I,) and coherence (|x|^2, |y|^2, Re, Im of
    conj(x) y) of rows x = 0, y = 1."""
    if mode == 'scalar':
        return np.abs(z) ** 2
    x, y = z[..., 0, :], z[..., 1, :]
    xx, yy = np.abs(x) ** 2, np.abs(y) ** 2
    if mode == 'stokes_i':
        return (xx + yy)[..., None, :]
    if mode == 'stokes':
        c = x * np.conj(y)
        return np.stack([xx + yy, xx - yy, 2 * c.real, -2 * c.imag], axis=-2)
    if mode == 'coherence':
        c = np.conj(x) * y
        return np.stack([xx, yy, c.real, c.imag], axis=-2)
    raise ValueError("unsupported mode %r" % (mode,))


def filterbank(x, f0, df, dm, nfft, nfine=1, mode='scalar', nint=1):
    """The operation on x [nchan, nb, ntime]: float64 [nchan nfine, P,
    ntime / (nfine nint)]."""
    z = fine_channels(x, f0, df, dm, nfft, nfine, nint)
    nchan = z.shape[0]
    d = detect(z, mode).reshape(nchan * nfine, -1, z.shape[-1])
    return d.reshape(d.shape[0], d.shape[1], -1, nint).sum(-1)
