"""Beamformer oracle (numpy).  TEST INFRASTRUCTURE -- see oracle/__init__.py.

matmul_ab: c = alpha a.b + beta c, the a.b form of bfLinAlgMatMul, restated
for the beamformer layout of the reference's test/test_linalg.py:136-151
(weights [chan, beam, K] times voltages [chan, K, time]) and any other
numpy.matmul-shaped product.  Integer-valued operands are summed exactly and
rounded once to complex64; anything else is summed in float64."""
import numpy as np


def _components(x, conj):
    """(re, im, is_integer) of a structured ci4/ci8/ci16 array or of a complex
    / real numpy array.  ci4 is decoded through oracle/unpack.py with the
    nibble order of a byte-reversed (big-endian) ci4 array: high nibble real,
    both two's complement, the convention of bf.DataType, bfFft and bfMap."""
    from oracle.unpack import unpack
    x = np.asarray(x)
    if x.dtype.names == ('re_im',):                       # ci4: one byte per element
        v = unpack(x['re_im'].reshape(x.shape + (1,)), 4, True, byte_reverse=True).reshape(x.shape + (2,)).astype(np.int64)
        re, im, integer = v[..., 0], v[..., 1], True
    elif x.dtype.names:
        re, im, integer = x['re'].astype(np.int64), x['im'].astype(np.int64), True
    else:
        x = np.asarray(x, np.complex128)
        re, im = x.real, x.imag
        integer = bool(np.all(re == np.round(re)) and np.all(im == np.round(im)) and
                       np.abs(re).max(initial=0) < 2 ** 31 and np.abs(im).max(initial=0) < 2 ** 31)
        if integer:
            re, im = re.astype(np.int64), im.astype(np.int64)
    return re, (-im if conj else im), integer


def matmul_ab(a, b, alpha=1.0, beta=0.0, c=None, conj_a=False, conj_b=False):
    """c = alpha a.b + beta c (batch dims broadcast as numpy.matmul), cf32.

    a and b are structured ci4 / ci8 / ci16 arrays or complex arrays; conj_a /
    conj_b conjugate them.  When both operands are integer-valued the product
    is summed exactly in int64 and rounded once to complex64, otherwise it is
    summed in float64.  alpha and beta are applied in float32 as the kernels do:
    alpha * s, then + beta * c."""
    ar, ai, ia = _components(a, conj_a)
    br, bi, ib = _components(b, conj_b)
    if ia and ib:
        # exact integer sums; float64 BLAS is exact too while every partial sum
        # stays below 2^53, and much faster than numpy's int64 matmul
        bound = 2 * max(np.abs(ar).max(initial=0), np.abs(ai).max(initial=0)) * \
            max(np.abs(br).max(initial=0), np.abs(bi).max(initial=0)) * ar.shape[-1]
        t = np.float64 if bound < 2 ** 53 else np.int64
        ar, ai, br, bi = ar.astype(t), ai.astype(t), br.astype(t), bi.astype(t)
        re = (np.matmul(ar, br) - np.matmul(ai, bi)).astype(np.int64)
        im = (np.matmul(ar, bi) + np.matmul(ai, br)).astype(np.int64)
        s = re.astype(np.float32) + 1j * im.astype(np.float32)
    else:
        ac = ar.astype(np.float64) + 1j * ai.astype(np.float64)
        bc = br.astype(np.float64) + 1j * bi.astype(np.float64)
        s = np.matmul(ac, bc)
    s = s.astype(np.complex64)
    out = np.float32(alpha) * s.real + 1j * (np.float32(alpha) * s.imag)
    out = out.astype(np.complex64)
    if beta != 0:
        c = np.asarray(c, np.complex64)
        out = ((out.real + np.float32(beta) * c.real) + 1j * (out.imag + np.float32(beta) * c.imag)).astype(np.complex64)
    return out
