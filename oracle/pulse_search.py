"""Boxcar pulse-search oracle (numpy, fp64).  TEST INFRASTRUCTURE -- see
oracle/__init__.py.

The semantics of bfPulseSearchExecute (include/bifrost_b200.h), restated with
cumsum prefix sums and two-pass mean / standard deviation:
  b_w[t] = sum_{k<w} x[t+k] for the nout = ntime - W + 1 starts t;
  mu_w, sigma_w: mean and population std of b_w over those starts;
  block j = starts [j decim, min((j+1) decim, nout)): per width the first
  argmax t_w of b_w, s_w = (b_w[t_w] - mu_w) / sigma_w (0 if sigma_w == 0);
  the block reports the first width with the largest s_w as
  (s_w, t_w - j decim, w).
"""
import numpy as np


def boxcars(x, widths):
    """b[..., wi, t] (fp64) for the nout starts that fit the widest width."""
    x = np.asarray(x, dtype=np.float64)
    ntime = x.shape[-1]
    nout = ntime - max(widths) + 1
    if nout < 1:
        raise ValueError("ntime must be >= the widest width")
    c = np.zeros(x.shape[:-1] + (ntime + 1,), np.float64)
    np.cumsum(x, axis=-1, out=c[..., 1:])
    return np.stack([c[..., w:w + nout] - c[..., :nout] for w in widths], axis=-2)


def snr(x, widths):
    """(b, s) with s[..., wi, t] = (b - mu_w) / sigma_w, 0 where sigma_w == 0."""
    b = boxcars(x, widths)
    mu = b.mean(axis=-1, keepdims=True)
    sd = np.sqrt(((b - mu) ** 2).mean(axis=-1, keepdims=True))
    with np.errstate(invalid='ignore', divide='ignore'):
        s = np.where(sd > 0, (b - mu) / np.where(sd > 0, sd, 1.), 0.)
    return b, s


def pulse_search(x, widths, decim):
    """out [..., nblk, 3] float32 of (snr, offset, width), plus the fp64 snr."""
    widths = [int(w) for w in widths]
    b, s = snr(x, widths)
    nout = b.shape[-1]
    nblk = -(-nout // decim)
    lead = b.shape[:-2]
    out = np.zeros(lead + (nblk, 3), np.float32)
    best = np.zeros(lead + (nblk,), np.float64)
    for j in range(nblk):
        lo, hi = j * decim, min((j + 1) * decim, nout)
        tw = np.argmax(b[..., lo:hi], axis=-1)                            # first max per width
        sw = np.take_along_axis(s[..., lo:hi], tw[..., None], -1)[..., 0]  # [..., nwidth]
        wi = np.argmax(sw, axis=-1)                                        # first best width
        best[..., j] = np.take_along_axis(sw, wi[..., None], -1)[..., 0]
        out[..., j, 0] = best[..., j]
        out[..., j, 1] = np.take_along_axis(tw, wi[..., None], -1)[..., 0]
        out[..., j, 2] = np.asarray(widths)[wi]
    return out, best
