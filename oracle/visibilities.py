"""Visibility layout conversions (numpy, float32).  TEST INFRASTRUCTURE -- see
oracle/__init__.py.

C[..., r, s] is the correlator's matrix over r = 2 i + p (station i, pol p),
valid for r >= s only; nothing here reads r < s.  Every output is one float32
add, subtract, multiplication by 0.5 or sign change of the inputs, in the
order written below, so it is the value the kernels of
bifrost_b200/csrc/visibilities.cu must produce bit for bit.

  fill_hermitian  out[r][s] = C[r][s] (r >= s), conj(C[s][r]) (r < s)
  to_storage      [..., nchan, nstand, 2, nstand, 2] -> [..., nbaseline, nchan, 4]
                  b = i (i + 1) / 2 + j, i >= j;  xy = conj(yx) when i == j;
                  I = xx + yy, Q = xx - yy, U = xy + yx, V = i (xy - yx)
  from_storage    xx = (I + Q) / 2, yy = (I - Q) / 2, xy = (U - i V) / 2,
                  yx = (U + i V) / 2, xy = conj(yx) when i == j; for i < j
                  out[i, p, j, q] = conj(C[j, q, i, p])
"""
import numpy as np


def _parts(z):
    return np.real(z).astype(np.float32), np.imag(z).astype(np.float32)


def _cplx(re, im):
    out = np.empty(np.shape(re), np.complex64)
    out.real, out.imag = re, im
    return out


def _conj(z):
    re, im = _parts(z)
    return _cplx(re, -im)


def _add(a, b):
    (ar, ai), (br, bi) = _parts(a), _parts(b)
    return _cplx(ar + br, ai + bi)


def _sub(a, b):
    (ar, ai), (br, bi) = _parts(a), _parts(b)
    return _cplx(ar - br, ai - bi)


def _half(a):
    re, im = _parts(a)
    return _cplx(np.float32(0.5) * re, np.float32(0.5) * im)


def _times_i(a):
    re, im = _parts(a)
    return _cplx(-im, re)


def fill_hermitian(c):
    """c: [..., n, n] complex64, lower triangle valid -> full Hermitian matrix."""
    c = np.asarray(c, np.complex64)
    n = c.shape[-1]
    out = np.empty_like(c)
    il = np.tril_indices(n)
    out[..., il[0], il[1]] = c[..., il[0], il[1]]
    iu = np.triu_indices(n, 1)
    out[..., iu[0], iu[1]] = _conj(c[..., iu[1], iu[0]])
    return out


def nbaseline(nstand):
    return nstand * (nstand + 1) // 2


def baselines(nstand):
    """(i, j) of every baseline b = i (i + 1) / 2 + j, in order of b."""
    i, j = np.tril_indices(nstand)       # row-major over the lower triangle: exactly b order
    return i, j


def to_storage(c):
    """c: [..., nchan, nstand, 2, nstand, 2] -> [..., nbaseline, nchan, 4]."""
    c = np.asarray(c, np.complex64)
    nstand = c.shape[-4]
    i, j = baselines(nstand)
    # [..., nchan, nbaseline] each
    xx = c[..., i, 0, j, 0]
    yx = c[..., i, 1, j, 0]
    yy = c[..., i, 1, j, 1]
    xy = _conj(yx)
    off = i != j                          # C[i, 0, i, 1] is above the diagonal
    xy[..., off] = c[..., i[off], 0, j[off], 1]
    stokes = np.stack([_add(xx, yy), _sub(xx, yy), _add(xy, yx), _times_i(_sub(xy, yx))], axis=-1)
    return np.ascontiguousarray(np.swapaxes(stokes, -2, -3))


def from_storage(s):
    """s: [..., nbaseline, nchan, 4] -> [..., nchan, nstand, 2, nstand, 2]."""
    s = np.asarray(s, np.complex64)
    nb, nchan = s.shape[-3], s.shape[-2]
    nstand = int(np.rint((np.sqrt(8 * nb + 1) - 1) / 2))
    assert nbaseline(nstand) == nb
    v = np.swapaxes(s, -2, -3)           # [..., nchan, nbaseline, 4]
    I, Q, U, V = (v[..., k] for k in range(4))
    i, j = baselines(nstand)
    xx = _half(_add(I, Q))
    yy = _half(_sub(I, Q))
    yx = _half(_add(U, _times_i(V)))
    xy = np.where(i == j, _conj(yx), _half(_sub(U, _times_i(V))))
    out = np.empty(s.shape[:-3] + (nchan, nstand, 2, nstand, 2), np.complex64)
    for (p, q), val in (((0, 0), xx), ((0, 1), xy), ((1, 0), yx), ((1, 1), yy)):
        out[..., i, p, j, q] = val
        off = i != j                      # mirror: out[j, q, i, p] = conj(C[i, p, j, q])
        out[..., j[off], q, i[off], p] = _conj(val[..., off])
    return out
