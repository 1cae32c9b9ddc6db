"""Generates tests/golden/ref_gpu_golden.npz: what the reference's own CUDA
library (oracle/_ref/libbifrost_ref.so, built by oracle/ref_build.sh) returns
for the inputs of the GPU parity tests of bfReduce, bfLinAlgMatMul (the
correlator form), bfFdmtExecute and bfQuantize.  The tests compare this
library's outputs with these stored ones, so they need neither the reference
tree nor its library.  Large outputs are kept as a fixed seeded sample of
their elements (`sample_index`) so that the file stays small.  Needs a GPU:

    bash oracle/ref_build.sh && python tests/golden/make_ref_gpu_golden.py OUT.npz

then copy OUT.npz to tests/golden/ref_gpu_golden.npz.
"""
import ctypes
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
PATH = os.path.join(HERE, 'ref_gpu_golden.npz')

# bfReduce: input a = rng.normal(size=shape), rng = default_rng(11) drawn in this order
REDUCE_CASES = [((4096, 256), 1, 4), ((4096, 256), 0, 8), ((4, 65536), 1, 4), ((20, 40, 60), 1, 5)]
REDUCE_OPS = ['sum', 'min', 'max', 'mean', 'pwrsum']
# correlator b^H.b over x[ntime, nchan, n] ci8, rng = default_rng(77) drawn in this order
LINALG_CASES = [(64, 3, 32), (512, 4, 512), (200, 2, 130)]
# FDMT (ntime, nchan, max_delay, dtype), rng = default_rng(7) drawn in this order
FDMT_CASES = [(2000, 256, 301, 'f32'), (1500, 100, 64, 'i8'), (4096, 512, 130, 'i8'), (333, 17, 40, 'u16')]
FDMT_SENTINEL = -999.0
# bfQuantize (odtype, nbit) x scale
QUANTIZE_CASES = [(o, b, s) for s in (1.0, 0.37)
                  for o, b in [('i4', 4), ('ci4', 4), ('i2', 2), ('ci2', 2), ('i1', 1), ('ci1', 1)]]
SAMPLE = 8192


def sample_index(size, key):
    """Fixed sample of flat indices of an output with `size` elements."""
    if size <= SAMPLE:
        return np.arange(size)
    return np.sort(np.random.default_rng(key).choice(size, SAMPLE, replace=False))


def reduce_key(ci, op):
    return 'reduce/%d/%s' % (ci, op)


def reduce_inputs():
    rng = np.random.default_rng(11)
    return [rng.normal(size=shape).astype(np.float32) for shape, _, _ in REDUCE_CASES]


def reduce_oshape(ci):
    shape, axis, n = REDUCE_CASES[ci]
    oshape = list(shape)
    oshape[axis] //= n
    return oshape


def linalg_inputs():
    ci8 = np.dtype([('re', np.int8), ('im', np.int8)])
    rng = np.random.default_rng(77)
    xs = []
    for shape in LINALG_CASES:
        x = np.empty(shape, dtype=ci8)
        x['re'] = rng.integers(-127, 128, size=shape)
        x['im'] = rng.integers(-127, 128, size=shape)
        xs.append(x)
    return xs


def linalg_lower(c):
    """Lower-triangle entries [nchan, n(n+1)/2] of a correlator output [nchan, n, n]."""
    il = np.tril_indices(c.shape[-1])
    return c[:, il[0], il[1]]


def fdmt_inputs():
    rng = np.random.default_rng(7)
    xs = []
    for ntime, nchan, md, dtype in FDMT_CASES:
        if dtype == 'f32':
            x = rng.normal(size=(nchan, ntime)).astype(np.float32)
        else:
            info = np.iinfo({'i8': np.int8, 'u16': np.uint16}[dtype])
            x = rng.integers(max(info.min, -127), min(info.max, 127) + 1, size=(nchan, ntime)).astype(info.dtype)
        xs.append(x)
    return xs


def quantize_input(nbit, cplx, n=4096 * 8 + 24):
    rng = np.random.default_rng(nbit * 2 + cplx)
    x = (rng.normal(size=n) * (4.0 if nbit == 4 else 1.0)).astype(np.float32)
    x[:8] = [0.5, 1.5, 2.5, -0.5, -1.5, 1e20, -1e20, 6.5]
    if cplx:
        x = (x[0::2] + 1j * x[1::2]).astype(np.complex64)
    return x


def quantize_key(odtype, scale):
    return 'quantize/%s/%g' % (odtype, scale)


def main(out_path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import bifrost_b200 as bf
    from bifrost_b200.libbifrost import _bf, _check
    import reflib
    ref = reflib.load()
    assert ref is not None, 'oracle/_ref/libbifrost_ref.so missing: run oracle/ref_build.sh'
    bf.device.set_device(0)
    store = {}

    codes = dict(sum=_bf.BF_REDUCE_SUM, min=_bf.BF_REDUCE_MIN, max=_bf.BF_REDUCE_MAX,
                 mean=_bf.BF_REDUCE_MEAN, pwrsum=_bf.BF_REDUCE_POWER_SUM)
    for ci, a in enumerate(reduce_inputs()):
        d_a = bf.asarray(a, space='cuda')
        for op in REDUCE_OPS:
            d_r = bf.empty(reduce_oshape(ci), 'f32', 'cuda')
            _check(ref.bfReduce(d_a.as_BFarray(), d_r.as_BFarray(), codes[op]))
            _check(ref.bfStreamSynchronize())
            out = np.asarray(d_r.copy('system')).ravel()
            store[reduce_key(ci, op)] = out[sample_index(out.size, 1000 * ci)]

    for ci, x in enumerate(linalg_inputs()):
        nchan, n = x.shape[1], x.shape[2]
        d_x = bf.asarray(x, space='cuda')
        d_c = bf.zeros((nchan, n, n), 'cf32', 'cuda')
        h = ctypes.c_void_p()
        _check(ref.bfLinAlgCreate(ctypes.byref(h)))
        _check(ref.bfLinAlgMatMul(h, 1.0, None, d_x.transpose((1, 0, 2)).as_BFarray(), 0.0, d_c.as_BFarray()))
        _check(ref.bfStreamSynchronize())
        _check(ref.bfLinAlgDestroy(h))
        low = linalg_lower(np.asarray(d_c.copy('system'))).ravel()
        store['linalg/%d' % ci] = low[sample_index(low.size, 2000 + ci)]

    for ci, x in enumerate(fdmt_inputs()):
        ntime, nchan, md, _ = FDMT_CASES[ci]
        f0, df = 1000., 400. / nchan
        d_in = bf.asarray(x, space='cuda')
        d_out = bf.asarray(np.full((md, ntime), FDMT_SENTINEL, np.float32), space='cuda')
        plan = ctypes.c_void_p()
        _check(ref.bfFdmtCreate(ctypes.byref(plan)))
        _check(ref.bfFdmtInit(plan, nchan, md, f0, df, -2.0, 2, None, None))
        _check(ref.bfFdmtExecute(plan, d_in.as_BFarray(), d_out.as_BFarray(), 0, None, None))
        _check(ref.bfStreamSynchronize())
        _check(ref.bfFdmtDestroy(plan))
        out = np.asarray(d_out.copy('system')).ravel()
        store['fdmt/%d' % ci] = out[sample_index(out.size, 3000 + ci)]

    for odtype, nbit, scale in QUANTIZE_CASES:
        cplx = odtype.startswith('c')
        x = quantize_input(nbit, cplx)
        nbyte = x.size * (2 if cplx else 1) * nbit // 8
        d_in = bf.asarray(x, space='cuda')
        d_raw = bf.asarray(np.zeros(nbyte, np.uint8), space='cuda')
        d_out = bf.ndarray(space='cuda', buffer=d_raw.ctypes.data, shape=x.shape, dtype=odtype)
        # (the reference's contiguity test rejects the byte strides of most
        # sub-byte arrays -- BF_STATUS_UNSUPPORTED_STRIDE: nothing is stored then)
        if ref.bfQuantize(d_in.as_BFarray(), d_out.as_BFarray(), float(scale)) == 0:
            bf.device.stream_synchronize()
            store[quantize_key(odtype, scale)] = np.asarray(d_raw.copy('system'))

    np.savez_compressed(out_path, **store)
    print('wrote', out_path, os.path.getsize(out_path), 'bytes,', len(store), 'arrays')


def load():
    return np.load(PATH)


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else PATH)
