"""bfVisibilities* and the convert_visibilities block (the reference's
python/bifrost/blocks/convert_visibilities.py and test/test_pipeline.py:225-336).

CPU: oracle/visibilities.py against first principles (C = X^H X from ci8
voltages, summed exactly), and the block's header contract.
GPU: every kernel bit-exact against the oracle over station counts 1..2100,
channel counts 1..129, 1 and 3 frames and padded strides, with the upper
triangle of every matrix input set to NaN (it must never be read) and a
sentinel in the padding of every output (it must survive); each case asserts
which kernel ran.  Then real correlator output, the reference's two pipeline
tests restated, and the status codes of every rejection."""
import ctypes
import re

import numpy as np
import pytest

import bifrost_b200 as bf
from bifrost_b200.libbifrost import _bf
from bifrost_b200.pipeline import Pipeline
from oracle import visibilities as ovis

CI8 = bf.DataType('ci8').as_numpy_dtype()
SENTINEL = np.complex64(1234.5 - 678.25j)


def gram(x):
    """x: ci8 [ntime, nchan, n] -> exact X^H X per channel, [nchan, n, n] float64 complex."""
    xr = np.moveaxis(x['re'].astype(np.float64), 0, 1)
    xi = np.moveaxis(x['im'].astype(np.float64), 0, 1)
    xt_r, xt_i = np.swapaxes(xr, -1, -2), np.swapaxes(xi, -1, -2)
    return (xt_r @ xr + xt_i @ xi) + 1j * (xt_r @ xi - xt_i @ xr)


def rand_ci8(rng, shape):
    x = np.empty(shape, CI8)
    x['re'] = rng.integers(-128, 128, size=shape)
    x['im'] = rng.integers(-128, 128, size=shape)
    return x


def lower_only(c):
    """Copy of [..., n, n] with NaN everywhere above the diagonal."""
    c = np.array(c, np.complex64)
    iu = np.triu_indices(c.shape[-1], 1)
    c[..., iu[0], iu[1]] = np.nan + 1j * np.nan
    return c


def stokes_direct(full, nstand):
    """Stokes of every baseline from a full Hermitian matrix, in float64."""
    f = full.reshape(full.shape[:-2] + (nstand, 2, nstand, 2))
    i, j = np.tril_indices(nstand)
    xx, xy, yx, yy = (f[..., i, p, j, q] for p, q in ((0, 0), (0, 1), (1, 0), (1, 1)))
    s = np.stack([xx + yy, xx - yy, xy + yx, 1j * (xy - yx)], axis=-1)
    return np.swapaxes(s, -2, -3)


# ---------------------------------------------------------------------- CPU
def test_oracle_against_first_principles():
    rng = np.random.default_rng(1)
    ntime, nchan, nstand = 16, 3, 7
    full = gram(rand_ci8(rng, (ntime, nchan, 2 * nstand)))      # |C| < 2^20: exact in fp32
    low = lower_only(full)
    np.testing.assert_array_equal(ovis.fill_hermitian(low), full.astype(np.complex64))
    m6 = low.reshape(nchan, nstand, 2, nstand, 2)
    sto = ovis.to_storage(m6)
    assert sto.shape == (nstand * (nstand + 1) // 2, nchan, 4)
    np.testing.assert_array_equal(sto, stokes_direct(full, nstand).astype(np.complex64))
    back = ovis.from_storage(sto).reshape(nchan, 2 * nstand, 2 * nstand)
    np.testing.assert_array_equal(back, ovis.fill_hermitian(low))
    # batch dims pass through
    np.testing.assert_array_equal(ovis.to_storage(np.stack([m6, m6]))[1], sto)


class Seq(object):
    def __init__(self, header):
        self.header = header


def matrix_header(nchan=4, nstand=5, npol=2, mode='lower'):
    return {'_tensor': {'dtype': 'cf32', 'shape': [-1, nchan, nstand, npol, nstand, npol],
                        'labels': ['time', 'freq', 'station_i', 'pol_i', 'station_j', 'pol_j'],
                        'scales': [[0, 0.04], [50e6, 25e3], None, None, None, None],
                        'units': ['s', 'Hz', None, ['X', 'Y'], None, ['X', 'Y']]},
            'name': 'vis', 'gulp_nframe': 1, 'matrix_fill_mode': mode}


def make_block(fmt):
    from bifrost_b200 import blocks
    with Pipeline():
        src = blocks.array_source(np.zeros((1, 4, 5, 2, 5, 2), np.complex64), matrix_header(), gulp_nframe=1)
        return blocks.convert_visibilities(src, fmt)


def test_block_header_contract():
    full = make_block('matrix').on_sequence(Seq(matrix_header()))
    t = full['_tensor']
    assert t['shape'] == [-1, 4, 5, 2, 5, 2] and t['labels'] == matrix_header()['_tensor']['labels']
    assert t['scales'] == matrix_header()['_tensor']['scales'] and full['matrix_fill_mode'] == 'hermitian'
    assert make_block('matrix').on_sequence(Seq(matrix_header(npol=1, mode='hermitian')))['_tensor']['shape'] == \
        [-1, 4, 5, 1, 5, 1]

    sto = make_block('storage').on_sequence(Seq(matrix_header()))
    t = sto['_tensor']
    assert 'matrix_fill_mode' not in sto and t['dtype'] == 'cf32'
    assert t['shape'] == [-1, 15, 4, 4] and t['labels'] == ['time', 'baseline', 'freq', 'stokes']
    assert t['scales'] == [[0, 0.04], None, [50e6, 25e3], None]
    assert t['units'] == ['s', None, 'Hz', ['I', 'Q', 'U', 'V']]

    back = make_block('matrix').on_sequence(Seq(sto))
    t = back['_tensor']
    assert t['shape'] == [-1, 4, 5, 2, 5, 2] and t['labels'] == matrix_header()['_tensor']['labels']
    assert t['scales'] == [[0, 0.04], [50e6, 25e3], None, None, None, None]
    assert t['units'] == ['s', 'Hz', None, ['X', 'Y'], None, ['X', 'Y']]
    assert back['matrix_fill_mode'] == 'hermitian'

    with pytest.raises(NotImplementedError):
        make_block('triangular').on_sequence(Seq(matrix_header()))
    with pytest.raises(NotImplementedError):
        make_block('storage').on_sequence(Seq(sto))
    other = matrix_header()
    other['_tensor']['labels'] = ['time', 'freq', 'station', 'pol', 'station', 'pol']
    with pytest.raises(NotImplementedError):
        make_block('matrix').on_sequence(Seq(other))
    for bad in (matrix_header(npol=1), matrix_header(mode=None), matrix_header(mode='upper')):
        with pytest.raises(ValueError):
            make_block('storage').on_sequence(Seq(bad))
    bad = dict(sto, _tensor=dict(sto['_tensor'], shape=[-1, 14, 4, 4]))        # not triangular
    with pytest.raises(ValueError):
        make_block('matrix').on_sequence(Seq(bad))
    bad = dict(sto, _tensor=dict(sto['_tensor'], shape=[-1, 15, 4, 1]))
    with pytest.raises(ValueError):
        make_block('matrix').on_sequence(Seq(bad))
    bad = matrix_header()
    bad['_tensor']['dtype'] = 'ci32'
    with pytest.raises(ValueError):
        make_block('matrix').on_sequence(Seq(bad))


# ---------------------------------------------------------------------- GPU
def short(name):
    m = re.search(r'(\w+)\(', name)
    return m.group(1) if m else name


def ran(fn):
    from kernel_trace import device_kernels
    return [short(k) for k in device_kernels(fn)]


def host(d):
    return np.asarray(d.copy('system'))


def same_bits(got, want):
    got, want = np.asarray(got, np.complex64), np.asarray(want, np.complex64)
    assert got.shape == want.shape
    bad = got.view(np.uint64) != want.view(np.uint64)
    assert not bad.any(), "%i of %i differ, first at %s: %r vs %r" % (
        bad.sum(), bad.size, np.argwhere(bad)[0], got[bad][0], want[bad][0])


def matrix_input(rng, ntime, nchan, nstand, padded):
    """Device [ntime, nchan, nstand, 2, nstand, 2] cf32 view with NaN above
    the diagonal (and in the padding), plus its host values."""
    n = 2 * nstand
    vals = (rng.normal(size=(ntime, nchan, n, n)) + 1j * rng.normal(size=(ntime, nchan, n, n))).astype(np.complex64)
    vals = lower_only(vals).reshape(ntime, nchan, nstand, 2, nstand, 2)
    if not padded:
        return bf.asarray(vals, space='cuda'), vals
    base = np.full((ntime, nchan + 2, nstand + 1, 2, nstand, 2), np.nan, np.complex64)
    base[:, 1:nchan + 1, :nstand] = vals
    d_base = bf.asarray(base, space='cuda')
    return d_base[:, 1:nchan + 1, :nstand], vals


def matrix_output(ntime, nchan, nstand, padded):
    """Device output view filled with the sentinel, its base, and the view's index."""
    if not padded:
        d = bf.asarray(np.full((ntime, nchan, nstand, 2, nstand, 2), SENTINEL), space='cuda')
        return d, d, np.s_[...]
    d_base = bf.asarray(np.full((ntime, nchan + 1, nstand + 1, 2, nstand, 2), SENTINEL), space='cuda')
    view = np.s_[:, :nchan, 1:]
    return d_base[view], d_base, view


def storage_output(ntime, nb, nchan, padded):
    if not padded:
        d = bf.asarray(np.full((ntime, nb, nchan, 4), SENTINEL), space='cuda')
        return d, d, np.s_[...]
    d_base = bf.asarray(np.full((ntime, nb + 1, nchan + 1, 4), SENTINEL), space='cuda')
    view = np.s_[:, 1:, :nchan]
    return d_base[view], d_base, view


def check_padding(got_base, view):
    pad = np.ones(got_base.shape, bool)
    pad[view] = False
    assert (got_base[pad] == SENTINEL).all()


def as_square(d, ntime, nchan, nstand):
    return d.reshape(ntime, nchan, 2 * nstand, 2 * nstand)


CASES = [  # (nstand, nchan, ntime, padded)
    (1, 1, 1, False), (1, 3, 3, True), (2, 129, 1, False), (2, 1, 3, True),
    (31, 3, 3, False), (32, 128, 1, True), (33, 129, 1, False), (33, 3, 3, True),
    (60, 128, 1, False), (60, 3, 3, True), (256, 3, 1, False), (256, 1, 3, True),
]


@pytest.mark.gpu
@pytest.mark.parametrize("nstand,nchan,ntime,padded", CASES + [(2100, 1, 1, False)])
def test_kernels_bit_exact(nstand, nchan, ntime, padded):
    rng = np.random.default_rng(nstand * 1000 + nchan * 10 + ntime)
    nb = nstand * (nstand + 1) // 2
    d_m, m = matrix_input(rng, ntime, nchan, nstand, padded)

    d_f, d_fbase, fview = matrix_output(ntime, nchan, nstand, padded)
    assert ran(lambda: bf.visibilities.fill_hermitian(as_square(d_m, ntime, nchan, nstand),
                                                      as_square(d_f, ntime, nchan, nstand))) == \
        ['vis_fill_hermitian_kernel']
    got = host(d_fbase)
    n = 2 * nstand
    same_bits(got[fview].reshape(ntime, nchan, n, n), ovis.fill_hermitian(m.reshape(ntime, nchan, n, n)))
    check_padding(got, fview)

    d_s, d_sbase, sview = storage_output(ntime, nb, nchan, padded)
    assert ran(lambda: bf.visibilities.to_storage(d_m, d_s)) == ['vis_to_storage_kernel']
    got = host(d_sbase)
    same_bits(got[sview], ovis.to_storage(m))
    check_padding(got, sview)
    del d_m, d_f, d_fbase

    # from_storage on general float values (the halving rounds)
    sto = (rng.normal(size=(ntime, nb, nchan, 4)) + 1j * rng.normal(size=(ntime, nb, nchan, 4))).astype(np.complex64)
    if padded:
        sbase = np.full((ntime, nb + 2, nchan + 1, 4), np.nan, np.complex64)
        sbase[:, 2:, 1:] = sto
        d_in = bf.asarray(sbase, space='cuda')[:, 2:, 1:]
    else:
        d_in = bf.asarray(sto, space='cuda')
    d_o, d_obase, oview = matrix_output(ntime, nchan, nstand, padded)
    assert ran(lambda: bf.visibilities.from_storage(d_in, d_o)) == ['vis_from_storage_kernel']
    got = host(d_obase)
    same_bits(got[oview], ovis.from_storage(sto))
    check_padding(got, oview)


@pytest.mark.gpu
def test_real_correlator_output():
    """ci8 -> LinAlg.matmul (lower triangle) -> fill_hermitian is X^H X exactly,
    and to_storage is its Stokes."""
    rng = np.random.default_rng(5)
    ntime, nchan, nstand = 64, 5, 40
    n = 2 * nstand
    x = rand_ci8(rng, (ntime, nchan, n))
    full = gram(x)                                                  # |C| < 2^22: exact
    d_x = bf.asarray(x, space='cuda')
    d_c = bf.asarray(np.full((nchan, n, n), np.nan, np.complex64), space='cuda')
    bf.linalg.LinAlg().matmul(1, None, d_x.transpose((1, 0, 2)), 0, d_c)
    d_f = bf.empty((nchan, n, n), 'cf32', 'cuda')
    bf.visibilities.fill_hermitian(d_c, d_f)
    np.testing.assert_array_equal(host(d_f), full.astype(np.complex64))
    d_s = bf.empty((nstand * (nstand + 1) // 2, nchan, 4), 'cf32', 'cuda')
    bf.visibilities.to_storage(d_c.reshape(nchan, nstand, 2, nstand, 2), d_s)
    np.testing.assert_array_equal(host(d_s), stokes_direct(full, nstand).astype(np.complex64))


def closed_form_input(ntime, nchan, nstand, npol):
    """CorrelateTestInputBlock of the reference (test/test_pipeline.py:66-72)."""
    i = np.arange(nstand * npol * 2) % 255 - 127
    x = np.empty((ntime, nchan, nstand, npol), dtype=CI8)
    x['re'] = i[0::2].reshape(nstand, npol)
    x['im'] = i[1::2].reshape(nstand, npol)
    return x


@pytest.mark.gpu
def test_pipeline_correlate_then_convert():
    """test/test_pipeline.py:225-336: correlate -> convert_visibilities('matrix')
    equals the closed form in full, upper half included, and correlate ->
    'storage' -> 'matrix' equals it too; both sequences carry the same header."""
    from bifrost_b200 import blocks
    nint, gulp, nchan, nstand, npol = 1000, 100, 128, 60, 2
    x = closed_form_input(2 * nint, nchan, nstand, npol)
    hdr = {'_tensor': {'dtype': 'ci8', 'shape': [-1, nchan, nstand, npol],
                       'labels': ['time', 'freq', 'station', 'pol'],
                       'scales': [[0, 1 / 25e3], [50e6, 25e3], None, None],
                       'units': ['s', 'Hz', None, ['X', 'Y']]},
           'name': 'corr', 'gulp_nframe': gulp}
    out = {'direct': [], 'storage': [], 'round_trip': []}
    seqs = {}

    def sink(key, b):
        blocks.callback_sink(b, lambda s: seqs.__setitem__(key, s.header),
                             lambda s: out[key].append(np.array(s.data.copy('system'))))

    with Pipeline() as p:
        src = blocks.array_source(x, hdr, gulp_nframe=gulp)
        b = blocks.copy(src, space='cuda')
        b = blocks.correlate(b, nint)
        sink('direct', blocks.convert_visibilities(b, 'matrix'))
        s = blocks.convert_visibilities(b, 'storage')
        sink('storage', s)
        sink('round_trip', blocks.convert_visibilities(s, 'matrix'))
        p.run()
    for key in ('direct', 'round_trip'):
        t = seqs[key]['_tensor']
        assert seqs[key]['matrix_fill_mode'] == 'hermitian'
        assert seqs[key]['gulp_nframe'] == seqs['storage']['gulp_nframe']
        assert t['shape'] == [-1, nchan, nstand, npol, nstand, npol] and t['dtype'] == 'cf32'
        assert t['labels'] == ['time', 'freq', 'station_i', 'pol_i', 'station_j', 'pol_j']
        assert t['scales'] == [[0, nint / 25e3], [50e6, 25e3], None, None, None, None]
        assert t['units'] == ['s', 'Hz', None, ['X', 'Y'], None, ['X', 'Y']]
    assert seqs['storage']['_tensor']['labels'] == ['time', 'baseline', 'freq', 'stokes']

    i = np.arange(nstand * npol * 2) % 255 - 127
    v = i[0::2] + 1j * i[1::2]
    expected = (nint * v[:, None].conj() * v[None, :]).astype(np.complex64)      # exact integers, rounded once
    expected = np.broadcast_to(expected.reshape(nstand, npol, nstand, npol), (1, nchan, nstand, npol, nstand, npol))
    direct = np.concatenate(out['direct'])
    assert direct.shape == (2,) + expected.shape[1:]
    for frame in direct:
        np.testing.assert_array_equal(frame, expected[0])
    round_trip = np.concatenate(out['round_trip'])
    np.testing.assert_allclose(round_trip, direct, rtol=1e-6, atol=1e-6 * np.abs(direct).max())
    storage = np.concatenate(out['storage'])
    same_bits(storage, ovis.to_storage(direct))


def bfa(shape, dtype='cf32', space='cuda'):
    return bf.empty(shape, dtype, space)


@pytest.mark.gpu
def test_status_codes():
    def st(fn, a, b):
        return fn(a.as_BFarray(), b.as_BFarray())
    fill, to, frm = _bf.bfVisibilitiesFillHermitian, _bf.bfVisibilitiesToStorage, _bf.bfVisibilitiesFromStorage
    m = bfa((2, 3, 4, 2, 4, 2))
    s = bfa((2, 10, 3, 4))
    sq = bfa((2, 3, 8, 8))
    assert st(to, m, s) == 0 and st(frm, s, bfa(m.shape)) == 0 and st(fill, sq, bfa(sq.shape)) == 0
    # dtype and space
    assert st(to, bfa(m.shape, 'cf64'), s) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    assert st(fill, sq, bfa(sq.shape, 'ci16')) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    assert st(frm, bfa(s.shape, space='system'), m) == _bf.BF_STATUS_UNSUPPORTED_SPACE
    # npol != 2, nstokes != 4, non-triangular / mismatched nbaseline, other shape mismatches
    assert st(to, bfa((2, 3, 4, 1, 4, 1)), s) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(to, m, bfa((2, 10, 3, 2))) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(to, m, bfa((2, 9, 3, 4))) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(frm, bfa((2, 15, 3, 4)), m) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(to, m, bfa((2, 10, 2, 4))) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(to, m, bfa((3, 10, 3, 4))) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(to, m, bfa((10, 3, 4))) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(to, bfa((2, 3, 4, 2, 5, 2)), s) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(fill, bfa((2, 3, 8, 7)), bfa((2, 3, 8, 7))) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(fill, sq, bfa((2, 3, 6, 6))) == _bf.BF_STATUS_INVALID_SHAPE
    # strides: non-unit innermost, a broadcast batch dim, a stride that is not a multiple of 8 B
    wide = bfa((2, 3, 8, 16))
    assert st(fill, wide[..., ::2], bfa(sq.shape)) == _bf.BF_STATUS_UNSUPPORTED_STRIDE
    a = sq.as_BFarray()
    a.strides[0] = 0
    assert fill(a, bfa(sq.shape).as_BFarray()) == _bf.BF_STATUS_UNSUPPORTED_STRIDE
    a = sq.as_BFarray()
    a.strides[1] += 4
    assert fill(a, bfa(sq.shape).as_BFarray()) == _bf.BF_STATUS_UNSUPPORTED_STRIDE
    # overlapping in and out
    assert st(fill, sq, sq) == _bf.BF_STATUS_INVALID_ARGUMENT
    big = bfa((2, 3, 8, 9))
    assert st(fill, big[..., :8], big[..., 1:]) == _bf.BF_STATUS_INVALID_ARGUMENT
    flat = bfa((2 * 3 * 4 * 2 * 4 * 2,))
    assert st(to, m, flat[:240].reshape(2, 10, 3, 4)) == 0
    assert st(to, flat.reshape(m.shape), flat[:240].reshape(2, 10, 3, 4)) == _bf.BF_STATUS_INVALID_ARGUMENT
    assert fill(None, sq.as_BFarray()) == _bf.BF_STATUS_INVALID_POINTER
    bf.device.stream_synchronize()
