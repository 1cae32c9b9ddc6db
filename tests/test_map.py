"""General bfMap (csrc/map_jit.cu): the reference's own test expressions
(test/test_map.py) and the examples of python/bifrost/map.py:96-112.

CPU: every expression must COMPILE for sm_90a (bfMapCompile needs no device)
in the form the reference would pick -- plain element references first,
callable views when the string indexes its arrays.  GPU: the numerics of the
reference's tests, value for value.
"""
import importlib

import numpy as np
import pytest

import bifrost_b200 as bf

bmap = importlib.import_module('bifrost_b200.map')


def _sys(shape, dtype, immutable=False):
    a = bf.ndarray(np.zeros(shape, dtype)) if not isinstance(dtype, str) else bf.empty(shape, dtype, 'system')
    if immutable:
        a.flags['WRITEABLE'] = False
    return a


COMPILE_CASES = [
    # func, data builder, kwargs, expected mode
    ("y = x+1", lambda: {'x': _sys((7,), np.int64, True), 'y': _sys((7,), np.int64)}, {}, 0),
    ("y = x*3", lambda: {'x': _sys((7,), np.int64, True), 'y': _sys((7,), np.int64)}, {}, 0),
    ("y = rint(pow(x, 2.f))", lambda: {'x': _sys((5, 5), np.int64, True), 'y': _sys((5, 5), np.int64)}, {}, 0),
    ("auto tmp = x; y = tmp*tmp", lambda: {'x': _sys((5,), np.int64, True), 'y': _sys((5,), np.int64)}, {}, 0),
    ("y = x; y += x", lambda: {'x': _sys((5,), np.int64, True), 'y': _sys((5,), np.int64)}, {}, 0),
    ("c = a*b", lambda: {'a': _sys((9,), np.float32), 'b': _sys((9, 1), np.float32), 'c': _sys((9, 9), np.float32)}, {}, 0),
    ("y = (x-m)/s", lambda: {'x': _sys((9,), np.int64), 'y': _sys((9,), np.int64), 'm': 1, 's': 3}, {}, 0),
    ("b = a(_-a.shape()/2)", lambda: {'a': _sys((5, 6, 7), np.int32), 'b': _sys((5, 6, 7), np.int32)}, {}, 1),
    ("y.assign(x.imag, x.real)", lambda: {'x': _sys((4, 4), np.complex64, True), 'y': _sys((4, 4), np.complex64)}, {}, 0),
    ("y = x*x.conj()", lambda: {'x': _sys((4,), np.complex64, True), 'y': _sys((4,), np.complex64)}, {}, 0),
    ("y = x.mag2()", lambda: {'x': _sys((4,), np.complex64, True), 'y': _sys((4,), np.complex64)}, {}, 0),
    ("y = 3*x", lambda: {'x': _sys((4,), np.complex64, True), 'y': _sys((4,), np.complex64)}, {}, 0),
    ("b(i) = a(i)", lambda: {'a': _sys((8,), 'ci4'), 'b': _sys((8,), 'cf32')}, dict(shape=(8,), axis_names=('i',)), 1),
    ("b(i) = a(i)", lambda: {'a': _sys((8,), 'ci4'), 'b': _sys((8,), 'ci4')}, dict(shape=(8,), axis_names=('i',)), 1),
    ("b(i) = a(i)", lambda: {'a': _sys((8,), 'ci8'), 'b': _sys((8,), 'cf32')}, dict(shape=(8,), axis_names=('i',)), 1),
    ("b(i) = a(i)", lambda: {'a': _sys((8,), 'ci16'), 'b': _sys((8,), 'ci16')}, dict(shape=(8,), axis_names=('i',)), 1),
    ("b(i) = a(i)", lambda: {'a': _sys((8,), 'ci32'), 'b': _sys((8,), 'cf32')}, dict(shape=(8,), axis_names=('i',)), 1),
    ("""
     auto x = a(_,0);
     auto y = a(_,1);
     b(_,0).assign(x.mag2(), y.mag2());
     b(_,1) = x*y.conj();
     """, lambda: {'a': _sys((9, 2), np.complex64), 'b': _sys((9, 2), np.complex64)}, dict(shape=(9,)), 1),
    ("b(i,j,k) = a(j,k,i)", lambda: {'a': _sys((5, 6, 7), np.int32), 'b': _sys((7, 5, 6), np.int32)},
     dict(shape=(7, 5, 6), axis_names=('i', 'j', 'k'), block_axes=('i', 'k')), 1),
    ("b(i,k) = a(i,j,k)", lambda: {'a': _sys((5, 6, 7), np.int32), 'b': _sys((5, 7), np.int32), 'j': 3},
     dict(shape=(5, 7), axis_names=('i', 'k')), 1),
    ("c(i,j) = a(i) * b(j)", lambda: {'c': _sys((4, 5), np.float32), 'a': _sys((4,), np.float32), 'b': _sys((5,), np.float32)},
     dict(axis_names=('i', 'j'), shape=(4, 5)), 1),
    ("a = c.real; b = c.imag", lambda: {'c': _sys((4,), np.complex64), 'a': _sys((4,), np.float32), 'b': _sys((4,), np.float32)}, {}, 0),
    ("c = pow(a, p)", lambda: {'c': _sys((4,), np.float32), 'a': _sys((4,), np.float32), 'p': 2.0}, {}, 0),
    # the hot-path blocks' own strings must also go through the general path
    ("b = beta * b + (b_type)a", lambda: {'a': _sys((4,), np.float32), 'b': _sys((4,), np.float32), 'beta': 0.5}, {}, 0),
    ("b = Complex<b_type>(a).mag2()", lambda: {'a': _sys((4,), 'ci8'), 'b': _sys((4,), np.float32)}, {}, 0),
    # extra_code: a helper at namespace scope
    ("y = twice(x)", lambda: {'x': _sys((4,), np.float32), 'y': _sys((4,), np.float32)},
     dict(extra_code="template<typename T> T twice(T v) { return v + v; }"), 0),
]


@pytest.mark.parametrize("func,data,kw,mode", COMPILE_CASES, ids=[c[0].strip().split('\n')[0][:28] + f"#{i}" for i, c in enumerate(COMPILE_CASES)])
def test_expressions_compile_for_sm_100a(func, data, kw, mode):
    assert bmap.compile_only(func, data(), **kw) == mode


def test_a_string_that_is_not_cxx_is_an_invalid_argument():
    with pytest.raises(Exception):
        bmap.compile_only("y = = x", {'x': _sys((4,), np.float32), 'y': _sys((4,), np.float32)})
    with pytest.raises(Exception):
        bmap.compile_only("y = x", {'x': _sys((4,), np.float32), 'y-': _sys((4,), np.float32)})


# ------------------------------------------------------------------ GPU ----
def _simple(x, funcstr, func):
    x_orig = x
    x = bf.asarray(x, 'cuda')
    y = bf.empty_like(x)
    x.flags['WRITEABLE'] = False
    for _ in range(3):
        bf.map(funcstr, {'x': x, 'y': y})
    xs = np.asarray(x.copy('system'))
    ys = np.asarray(y.copy('system'))
    np.testing.assert_equal(ys, func(xs if isinstance(x_orig, bf.ndarray) else x_orig))


def _simple_funcs(x):
    _simple(x, "y = x+1", lambda x: x + 1)
    _simple(x, "y = x*3", lambda x: x * 3)
    _simple(x, "y = rint(pow(x, 2.f))", lambda x: x ** 2)
    _simple(x, "auto tmp = x; y = tmp*tmp", lambda x: x * x)
    _simple(x, "y = x; y += x", lambda x: x + x)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(7919,), (89, 89), (23, 23, 23)])
def test_gpu_simple(shape):
    rng = np.random.default_rng(1234)
    _simple_funcs(rng.integers(0, 256, size=shape))


@pytest.mark.gpu
def test_gpu_simple_padded():
    rng = np.random.default_rng(1)
    x = bf.asarray(rng.integers(0, 256, size=(89, 89)), space='cuda')
    _simple_funcs(x[:, 1:])
    x = bf.asarray(rng.integers(0, 256, size=(23, 23, 23)), space='cuda')
    _simple_funcs(x[:, :, 1:])


@pytest.mark.gpu
def test_gpu_broadcast_scalar_manydim():
    n = 89
    a = bf.asarray(np.arange(n).astype(np.float32), space='cuda')
    b = a[:, None]
    c = bf.empty((n, n), 'f32', 'cuda')
    bf.map("c = a*b", data={'a': a, 'b': b, 'c': c})
    ah = np.arange(n).astype(np.float32)
    np.testing.assert_equal(np.asarray(c.copy('system')), ah * ah[:, None])
    x = bf.asarray(np.random.default_rng(2).integers(1, 256, size=7919), space='cuda')
    y = bf.empty_like(x)
    bf.map("y = (x-m)/s", data={'x': x, 'y': y, 'm': 1, 's': 3})
    np.testing.assert_equal(np.asarray(y.copy('system')), (np.asarray(x.copy('system')) - 1) // 3)
    known = np.arange(3 ** 8).reshape([3] * 8).astype(np.float32)
    a = bf.asarray(known, space='cuda')[:, :, :, :, :2, :, :, :]
    b = bf.empty_like(a)
    bf.map("b = a+1", data={'a': a, 'b': b})
    np.testing.assert_equal(np.asarray(b.copy('system')), known[:, :, :, :, :2] + 1)


@pytest.mark.gpu
def test_gpu_shift_and_explicit_indexing():
    rng = np.random.default_rng(3)
    ah = rng.integers(0, 65536, size=(55, 66, 77)).astype(np.int32)
    a = bf.asarray(ah, space='cuda')
    b = bf.empty_like(a)
    bf.map("b = a(_-a.shape()/2)", data={'a': a, 'b': b})
    np.testing.assert_equal(np.asarray(b.copy('system')), np.fft.fftshift(ah))
    b = bf.empty((77, 55, 66), 'i32', 'cuda')
    bf.map("b(i,j,k) = a(j,k,i)", shape=b.shape, axis_names=('i', 'j', 'k'), data={'a': a, 'b': b},
           block_shape=(64, 4), block_axes=('i', 'k'))
    np.testing.assert_equal(np.asarray(b.copy('system')), ah.transpose([2, 0, 1]))
    b = bf.empty((55, 77), 'i32', 'cuda')
    bf.map("b(i,k) = a(i,j,k)", shape=b.shape, axis_names=('i', 'k'), data={'a': a, 'b': b, 'j': 11})
    np.testing.assert_equal(np.asarray(b.copy('system')), ah[:, 11, :])


@pytest.mark.gpu
def test_gpu_complex_float():
    rng = np.random.default_rng(4)
    n = 89
    x = (rng.integers(-127, 128, size=(n, n)) + 1j * rng.integers(-127, 128, size=(n, n))).astype(np.complex64)
    _simple(x, "y.assign(x.imag, x.real)", lambda x: x.imag + 1j * x.real)
    _simple(x, "y = x*x.conj()", lambda x: x * x.conj())
    _simple(x, "y = x.mag2()", lambda x: x * x.conj())
    _simple(x, "y = 3*x", lambda x: 3 * x)


@pytest.mark.gpu
@pytest.mark.parametrize("in_dtype", ['ci4', 'ci8', 'ci16', 'ci32'])
def test_gpu_complex_integer(in_dtype):
    n = 7919
    rng = np.random.default_rng(5)
    if in_dtype == 'ci4':
        raw = rng.integers(0, 256, size=n, dtype=np.uint8)
        re = (raw.view(np.int8) >> 4).astype(np.float32)
        im = ((raw << 4).view(np.int8) >> 4).astype(np.float32)
        a = bf.ndarray(raw.view(bf.DataType('ci4').as_numpy_dtype()), dtype='ci4').copy('cuda')
    else:
        nbit = int(in_dtype[2:])
        h = np.zeros(n, bf.DataType(in_dtype).as_numpy_dtype())
        h['re'] = rng.integers(-100, 100, size=n)
        h['im'] = rng.integers(-100, 100, size=n)
        re, im = h['re'].astype(np.float32), h['im'].astype(np.float32)
        a = bf.ndarray(h, dtype=in_dtype).copy('cuda')
    for out_dtype in (in_dtype, 'cf32'):
        b = bf.empty((n,), out_dtype, 'cuda')
        bf.map('b(i) = a(i)', {'a': a, 'b': b}, shape=a.shape, axis_names=('i',))
        out = np.asarray(b.copy('system'))
        if out_dtype == 'cf32':
            np.testing.assert_equal(out, re + 1j * im)
        elif in_dtype == 'ci4':
            np.testing.assert_equal(out.view(np.uint8), raw)
        else:
            np.testing.assert_equal(out['re'], h['re'])
            np.testing.assert_equal(out['im'], h['im'])


@pytest.mark.gpu
def test_gpu_polarisation_products():
    rng = np.random.default_rng(6)
    n = 89
    ah = (rng.integers(-127, 128, size=(n, 2)) + 1j * rng.integers(-127, 128, size=(n, 2))).astype(np.complex64)
    a = bf.asarray(ah, space='cuda')
    b = bf.empty_like(a)
    bf.map('''
        auto x = a(_,0);
        auto y = a(_,1);
        b(_,0).assign(x.mag2(), y.mag2());
        b(_,1) = x*y.conj();
        ''', shape=b.shape[:-1], data={'a': a, 'b': b})
    gold = np.empty_like(ah)
    mag2 = lambda z: z.real * z.real + z.imag * z.imag
    gold[..., 0] = mag2(ah[..., 0]) + 1j * mag2(ah[..., 1])
    gold[..., 1] = ah[..., 0] * ah[..., 1].conj()
    np.testing.assert_equal(np.asarray(b.copy('system')), gold)


@pytest.mark.gpu
def test_gpu_general_path_agrees_with_the_compiled_hot_path_kernels(monkeypatch):
    """detect 'scalar' and accumulate through NVRTC (BFB_MAP_JIT_ONLY) == the fixed kernels."""
    rng = np.random.default_rng(7)
    h = np.zeros(5000, bf.DataType('ci8').as_numpy_dtype())
    h['re'] = rng.integers(-127, 128, size=5000)
    h['im'] = rng.integers(-127, 128, size=5000)
    a = bf.ndarray(h, dtype='ci8').copy('cuda')
    outs = []
    for jit in (False, True):
        if jit:
            monkeypatch.setenv('BFB_MAP_JIT_ONLY', '1')
        b = bf.zeros((5000,), 'f32', 'cuda')
        bf.map("b = Complex<b_type>(a).mag2()", {'a': a, 'b': b})
        acc = bf.asarray(np.arange(5000, dtype=np.float32), space='cuda')
        bf.map("b = beta * b + (b_type)a", {'a': b, 'b': acc, 'beta': 0.5})
        outs.append((np.asarray(b.copy('system')), np.asarray(acc.copy('system'))))
    np.testing.assert_equal(outs[0][0], outs[1][0])
    np.testing.assert_equal(outs[0][1], outs[1][1])
    bf.clear_map_cache()
