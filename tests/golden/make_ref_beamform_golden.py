"""Generates tests/golden/ref_beamform_golden.npz: what the reference's own
bfLinAlgMatMul (oracle/_ref/libbifrost_ref.so, built by oracle/ref_build.sh;
its bf_cgemm_TN_smallM kernel) returns for the beamformer layout of the
reference's test/test_linalg.py:136-151,

    b[chan, beam, time] = sum_k w[chan, beam, k] x[chan, k, time]
    a = w.transpose(1, 0, 2) (cf32), b = x.transpose(1, 2, 0) (ci4 / ci8),

over that test's shapes (nbeam 1/5/12, nstand 16/64/256 x 2 pols, ntime
1/8/512, nchan 1/3/10) with ci4 and ci8 voltages and integer-valued cf32
weights, small enough that every fp32 sum is exact.  Inputs are regenerated
from `case_inputs`; each output is kept as a fixed seeded sample of its
elements so that the file stays small.  Needs a GPU:

    bash oracle/ref_build.sh && python tests/golden/make_ref_beamform_golden.py OUT.npz

then copy OUT.npz to tests/golden/ref_beamform_golden.npz.
"""
import ctypes
import itertools
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
PATH = os.path.join(HERE, 'ref_beamform_golden.npz')

CASES = list(itertools.product(('ci4', 'ci8'), (1, 5, 12), (16, 64, 256), (1, 8, 512), (1, 3, 10)))
SAMPLE = 256


def key(ci):
    xk, nbeam, nstand, ntime, nchan = CASES[ci]
    return 'beamform/%s/nbeam%d/nstand%d/ntime%d/nchan%d' % (xk, nbeam, nstand, ntime, nchan)


def case_inputs(ci):
    """(x [ntime, nchan, K] structured ci4 / ci8, w [nbeam, nchan, K] complex64).
    ci8 voltages span -127..127, ci4 -8..7; |w| <= 64 keeps sum_k |w| |x| < 2^24."""
    import bifrost_b200 as bf
    xk, nbeam, nstand, ntime, nchan = CASES[ci]
    K = 2 * nstand
    rng = np.random.default_rng(5000 + ci)
    if xk == 'ci8':
        x = np.empty((ntime, nchan, K), bf.DataType('ci8').as_numpy_dtype())
        x['re'] = rng.integers(-127, 128, size=x.shape)
        x['im'] = rng.integers(-127, 128, size=x.shape)
    else:
        x = rng.integers(0, 256, size=(ntime, nchan, K), dtype=np.uint8).view(bf.DataType('ci4').as_numpy_dtype())
    w = (rng.integers(-64, 65, size=(nbeam, nchan, K)) +
         1j * rng.integers(-64, 65, size=(nbeam, nchan, K))).astype(np.complex64)
    return x, w


def sample_index(size, ci):
    if size <= SAMPLE:
        return np.arange(size)
    return np.sort(np.random.default_rng(9000 + ci).choice(size, SAMPLE, replace=False))


def main(out_path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.dirname(HERE))
    import bifrost_b200 as bf
    from bifrost_b200.libbifrost import _check
    import reflib
    from oracle import beamform as obeamform
    ref = reflib.load()
    assert ref is not None, 'oracle/_ref/libbifrost_ref.so missing: run oracle/ref_build.sh'
    store = {}
    for ci in range(len(CASES)):
        xk, nbeam, nstand, ntime, nchan = CASES[ci]
        x, w = case_inputs(ci)
        d_x = bf.asarray(bf.ndarray(x, dtype=xk), space='cuda')
        d_w = bf.asarray(w, space='cuda')
        d_c = bf.zeros((nchan, nbeam, ntime), 'cf32', 'cuda')
        h = ctypes.c_void_p()
        _check(ref.bfLinAlgCreate(ctypes.byref(h)))
        st = ref.bfLinAlgMatMul(h, 1.0, d_w.transpose((1, 0, 2)).as_BFarray(),
                                d_x.transpose((1, 2, 0)).as_BFarray(), 0.0, d_c.as_BFarray())
        _check(ref.bfStreamSynchronize())
        _check(ref.bfLinAlgDestroy(h))
        assert st == 0, (key(ci), st)
        got = np.asarray(d_c.copy('system')).ravel()
        store[key(ci)] = got[sample_index(got.size, ci)]
        want = obeamform.matmul_ab(w.transpose(1, 0, 2), x.transpose(1, 2, 0)).ravel()
        verdict = 'equals the oracle' if np.array_equal(got, want) else 'DIFFERS from the oracle'
        if xk == 'ci4' and not np.array_equal(got, want):
            raw = x['re_im']
            xs = ((raw & 0xF) << 4 | raw >> 4).astype(np.uint8).view(x.dtype)
            swapped = obeamform.matmul_ab(w.transpose(1, 0, 2), xs.transpose(1, 2, 0)).ravel()
            verdict += ' (nibble-swapped oracle: %s)' % ('equal' if np.array_equal(got, swapped) else 'differs')
        print(key(ci), verdict, flush=True)
    np.savez_compressed(out_path, **store)


def load():
    return np.load(PATH)


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else PATH)
