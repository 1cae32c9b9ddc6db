"""bfLinAlgCorrelateToStorage, LinAlg.correlate_to_storage, correlate(...,
output='storage') and the block_scope(fuse=True) swap of correlate ->
convert_visibilities('storage').

The call is defined as bfLinAlgMatMul(1, NULL, x, 0, C) followed by
bfVisibilitiesToStorage(C, vis), bit for bit.  Every GPU case compares the
output as uint64 with oracle/visibilities.to_storage(oracle/linalg.correlate(x))
and with those two device calls, and asserts which kernels ran: the fused
corr_storage_tc_kernel<WIDE> (ci8 the tensor-core correlator takes in one
pass), or the matrix correlator into the handle's workspace followed by
vis_to_storage_kernel (everything else).

CPU: the storage-output block's header against convert_visibilities', the
fuse swap and the cases it must leave alone, and a no-spill sm_90a build."""
import os
import re
import subprocess

import numpy as np
import pytest

import bifrost_b200 as bf
from bifrost_b200 import blocks
from bifrost_b200.blocks.testing import NumpySourceBlock, _Reader
from bifrost_b200.libbifrost import _bf
from bifrost_b200.linalg import LinAlg
from bifrost_b200.pipeline import Pipeline
from oracle import linalg as olinalg
from oracle import visibilities as ovis

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CI8 = bf.DataType('ci8').as_numpy_dtype()
CI16 = bf.DataType('ci16').as_numpy_dtype()
SENTINEL = np.complex64(1234.5 - 678.25j)


class Seq(object):
    def __init__(self, header):
        self.header = header


def volt_header(nchan, nstand, gulp=None, scales=True, units=True):
    t = {'dtype': 'ci8', 'shape': [-1, nchan, nstand, 2], 'labels': ['time', 'freq', 'station', 'pol']}
    if scales:
        t['scales'] = [[0, 1 / 25e3], [50e6, 25e3], None, None]
    if units:
        t['units'] = ['s', 'Hz', None, ['X', 'Y']]
    hdr = {'_tensor': t, 'name': 'volts'}
    if gulp is not None:
        hdr['gulp_nframe'] = gulp
    return hdr


# ---------------------------------------------------------------------- CPU
@pytest.mark.parametrize("scales,units", [(True, True), (False, False), (True, False)])
@pytest.mark.parametrize("gulp,nint", [(None, 1), (1, 4), (4, 12), (10, 10), (20, 10)])
def test_storage_header_equals_convert_visibilities(scales, units, gulp, nint):
    hdr = volt_header(3, 5, gulp, scales, units)
    with Pipeline():
        src = blocks.array_source(np.zeros((1, 3, 5, 2), CI8), hdr, gulp_nframe=1)
        mat = blocks.correlate(src, nint)
        conv = blocks.convert_visibilities(mat, 'storage')
        sto = blocks.correlate(src, nint, output='storage')
    want = conv.on_sequence(Seq(mat.on_sequence(Seq(hdr))))
    got = sto.on_sequence(Seq(hdr))
    assert got == want
    assert 'matrix_fill_mode' not in got and got['_tensor']['shape'] == [-1, 15, 3, 4]
    # the matrix output is what it was
    assert mat.on_sequence(Seq(hdr))['matrix_fill_mode'] == 'lower'


def test_storage_output_needs_two_pols_and_a_known_output():
    hdr = volt_header(3, 5)
    hdr['_tensor']['shape'] = [-1, 3, 5, 1]
    with Pipeline():
        src = blocks.array_source(np.zeros((1, 3, 5, 1), CI8), hdr, gulp_nframe=1)
        sto = blocks.correlate(src, 1, output='storage')
        with pytest.raises(ValueError):
            blocks.correlate(src, 1, output='triangle')
    with pytest.raises(ValueError):
        sto.on_sequence(Seq(hdr))


def build_chain(fuse_corr=True, fuse_conv=True, fmt='storage', second_reader=False, view=False):
    from bifrost_b200 import block_scope, block_view
    with Pipeline() as p:
        src = blocks.array_source(np.zeros((4, 3, 5, 2), CI8), volt_header(3, 5, 2), gulp_nframe=2)
        with block_scope(fuse=fuse_corr, gpu=0, core=1):
            c = blocks.correlate(src, 4, gulp_nframe=2)
        if view:
            c = block_view(c, lambda h: h)
        with block_scope(fuse=fuse_conv):
            v = blocks.convert_visibilities(c, fmt)
        if second_reader:
            blocks.callback_sink(c)
        sink = blocks.callback_sink(v)
    return p, src, sink


def test_fuse_swaps_correlate_then_storage():
    from bifrost_b200.blocks.correlate import CorrelateBlock
    p, src, sink = build_chain()
    p._fuse_chains()
    kinds = [type(b).__name__ for b in p.blocks]
    assert 'ConvertVisibilitiesBlock' not in kinds and kinds.count('CorrelateBlock') == 1
    corr = [b for b in p.blocks if isinstance(b, CorrelateBlock)][0]
    assert corr.output == 'storage' and corr.nframe_per_integration == 4
    assert (corr.gulp_nframe, corr.gpu, corr.core) == (2, 0, 1)
    assert src.orings[0].consumers == [corr] and corr.irings == [src.orings[0]]
    assert corr.orings[0].consumers == [sink] and corr.orings[0].owner is corr
    assert sink.irings == [corr.orings[0]]


@pytest.mark.parametrize("kw", [dict(fuse_corr=False), dict(fuse_conv=False), dict(fmt='matrix'),
                                dict(second_reader=True), dict(view=True)])
def test_fuse_leaves_other_chains_alone(kw):
    p, src, sink = build_chain(**kw)
    before = list(p.blocks)
    p._fuse_chains()
    assert p.blocks == before
    assert all(getattr(b, 'output', 'matrix') == 'matrix' for b in p.blocks)


def test_kernel_compiles_without_spills(tmp_path):
    """corr_storage_tc_kernel, both WIDE instantiations: sm_90a, no spills."""
    src = os.path.join(ROOT, 'bifrost_b200', 'csrc')
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    out = subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17',
                          '-I' + os.path.join(ROOT, 'include'), '-I' + src, '--expt-relaxed-constexpr',
                          '-Xptxas', '-v', '-c', os.path.join(src, 'linalg.cu'), '-o', str(tmp_path / 'l.o')],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    # ptxas prints each entry's 'Compiling entry function' line, then its spill line
    stats, entry = {}, None
    for line in out.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            entry = m.group(1)
        elif entry and 'spill stores' in line:
            stats[entry] = line
    fused = {k: v for k, v in stats.items() if 'corr_storage_tc_kernel' in k}
    assert len(fused) == 2, list(stats)
    assert all(' 0 bytes spill stores, 0 bytes spill loads' in v for v in fused.values()), fused


# ---------------------------------------------------------------------- GPU
def short(name):
    """'void bfb::corr_storage_tc_kernel<false>(...)' -> 'corr_storage_tc_kernel<false>'."""
    m = re.search(r'(\w+)(<[^()]*>)?\(', name)
    return m.group(1) + (m.group(2) or '') if m else name


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


def full_range_ci8(rng, shape):
    """Uniform over [-128, 127], -128 forced into whole rows (as the correlator edge tests)."""
    x = np.empty(shape, dtype=CI8)
    x['re'] = rng.integers(-128, 128, size=shape)
    x['im'] = rng.integers(-128, 128, size=shape)
    x['re'][3::5] = -128
    x['re'][..., 0] = -128
    x['im'][..., 0] = -128
    return x


def oracle_storage(u, nstand):
    """u: [nchan, ntime, n] (structured ints or complex) -> [nbaseline, nchan, 4]."""
    c = olinalg.correlate(u)
    return ovis.to_storage(c.reshape(c.shape[0], nstand, 2, nstand, 2))


def storage_view(nb, nchan, padded, fill):
    """Device vis [nb, nchan, 4], optionally a view of a padded buffer; its base and index."""
    if not padded:
        d = bf.asarray(np.full((nb, nchan, 4), fill, np.complex64), space='cuda')
        return d, d, np.s_[...]
    d_base = bf.asarray(np.full((nb + 1, nchan + 2, 4), fill, np.complex64), space='cuda')
    view = np.s_[1:, 1:nchan + 1]
    return d_base[view], d_base, view


def two_calls(la, xv, nchan, nstand):
    n = 2 * nstand
    d_c = bf.empty((nchan, n, n), 'cf32', 'cuda')
    d_s = bf.empty((nstand * (nstand + 1) // 2, nchan, 4), 'cf32', 'cuda')
    la.matmul(1, None, xv, 0, d_c)
    bf.visibilities.to_storage(d_c.reshape(nchan, nstand, 2, nstand, 2), d_s)
    return host(d_s)


def oracle_equal(got, want, conj):
    """Bitwise, except that with a conjugated input the correlator negates an
    exact zero imaginary part into -0 where the oracle has +0 (adding 0 makes
    both +0); the device-to-device comparison stays fully bitwise."""
    if conj:
        got, want = got + np.complex64(0), want + np.complex64(0)
    same_bits(got, want)


def run_case(la, xv, u, nchan, nstand, want_kernels, padded=False, conj=False):
    nb = nstand * (nstand + 1) // 2
    d_v, d_base, view = storage_view(nb, nchan, padded, np.complex64(np.nan + 1j * np.nan) if not padded
                                     else SENTINEL)
    names = ran(lambda: la.correlate_to_storage(xv, d_v))
    assert names == want_kernels, names
    got = host(d_base)
    if padded:
        pad = np.ones(got.shape, bool)
        pad[view] = False
        assert (got[pad] == SENTINEL).all()
    got = got[view]
    assert not np.isnan(got).any()
    oracle_equal(got, oracle_storage(u, nstand), conj)
    same_bits(got, two_calls(la, xv, nchan, nstand))


FUSED = 'corr_storage_tc_kernel<false>'
# (nstand, nchan, ntime): every nstand, ntime and nchan of the sweep at least
# once, without the cross product (the host oracle of 352 x 129 x 640 alone
# takes minutes)
FUSED_CASES = [
    (8, 3, 1), (8, 129, 64), (12, 1, 65), (12, 3, 640), (28, 129, 63), (32, 3, 65), (32, 1, 640),
    (36, 3, 64), (64, 129, 1), (64, 3, 640), (100, 1, 63), (100, 3, 640), (128, 3, 65), (176, 1, 640),
    (176, 3, 63), (256, 3, 64), (256, 1, 640), (352, 1, 640), (352, 3, 65),
]


@pytest.mark.gpu
@pytest.mark.parametrize("nstand,nchan,ntime", FUSED_CASES)
def test_fused_bit_exact(nstand, nchan, ntime):
    rng = np.random.default_rng(nstand * 10000 + nchan * 100 + ntime)
    x = full_range_ci8(rng, (ntime, nchan, 2 * nstand))
    xv = bf.asarray(x, space='cuda').transpose((1, 0, 2))
    run_case(LinAlg(), xv, np.transpose(x, (1, 0, 2)), nchan, nstand, [FUSED], padded=(nchan == 3))


@pytest.mark.gpu
def test_fused_wide_epilogue():
    """70000 samples: pair sums leave int32, the 64-bit epilogue runs (WIDE)."""
    rng = np.random.default_rng(3)
    nstand, nchan, ntime = 8, 2, 70000
    x = full_range_ci8(rng, (ntime, nchan, 2 * nstand))
    xv = bf.asarray(x, space='cuda').transpose((1, 0, 2))
    run_case(LinAlg(), xv, np.transpose(x, (1, 0, 2)), nchan, nstand, ['corr_storage_tc_kernel<true>'])


@pytest.mark.gpu
def test_fused_conjugated_view():
    rng = np.random.default_rng(4)
    nstand, nchan, ntime = 40, 3, 100
    x = full_range_ci8(rng, (ntime, nchan, 2 * nstand))
    xv = bf.asarray(x, space='cuda').transpose((1, 0, 2)).conj()
    u = np.conj(np.transpose(x['re'] + 1j * x['im'].astype(np.float64), (1, 0, 2)))
    run_case(LinAlg(), xv, u, nchan, nstand, [FUSED], padded=True, conj=True)


def workspace_kernels(simt=True):
    return ['corr_simt_kernel' if simt else 'corr_tc_kernel', 'vis_to_storage_kernel']


def ran_short(la, xv, d_v):
    return [re.sub(r'<.*', '', k) for k in ran(lambda: la.correlate_to_storage(xv, d_v))]


def int_complex(rng, shape, lim, dtype):
    """Integer-valued samples small enough that every float sum is exact."""
    re_, im_ = rng.integers(-lim, lim + 1, size=shape), rng.integers(-lim, lim + 1, size=shape)
    if dtype == 'cf32':
        return (re_ + 1j * im_).astype(np.complex64)
    x = np.empty(shape, CI16)
    x['re'], x['im'] = re_, im_
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ['ci16', 'cf32'])
def test_workspace_float_inputs(dtype):
    rng = np.random.default_rng(5)
    nstand, nchan, ntime = 20, 3, 50
    x = int_complex(rng, (ntime, nchan, 2 * nstand), 300, dtype)
    xv = bf.asarray(x, space='cuda').transpose((1, 0, 2))
    la = LinAlg()
    d_v, d_base, view = storage_view(nstand * (nstand + 1) // 2, nchan, True, SENTINEL)
    assert ran_short(la, xv, d_v) == workspace_kernels()
    got = host(d_base)
    same_bits(got[view], oracle_storage(np.transpose(x, (1, 0, 2)), nstand))
    same_bits(got[view], two_calls(la, xv, nchan, nstand))
    pad = np.ones(got.shape, bool)
    pad[view] = False
    assert (got[pad] == SENTINEL).all()


def check_workspace(la, xv, u, nchan, nstand, kernels, conj=False):
    d_v = bf.asarray(np.full((nstand * (nstand + 1) // 2, nchan, 4), np.nan, np.complex64), space='cuda')
    assert ran_short(la, xv, d_v) == kernels
    got = host(d_v)
    oracle_equal(got, oracle_storage(u, nstand), conj)
    same_bits(got, two_calls(la, xv, nchan, nstand))


@pytest.mark.gpu
def test_workspace_channel_stride_not_16_bytes():
    """nstand = 10: the channel stride of the [time, chan, n] frame is 40 B."""
    rng = np.random.default_rng(6)
    nstand, nchan, ntime = 10, 3, 70
    x = full_range_ci8(rng, (ntime, nchan, 2 * nstand))
    check_workspace(LinAlg(), bf.asarray(x, space='cuda').transpose((1, 0, 2)), np.transpose(x, (1, 0, 2)),
                    nchan, nstand, workspace_kernels())


@pytest.mark.gpu
def test_workspace_misaligned_base():
    rng = np.random.default_rng(7)
    nstand, nchan, ntime = 16, 2, 90
    n = 2 * nstand
    x = full_range_ci8(rng, (ntime, nchan, n + 8))
    xv = bf.asarray(x, space='cuda')[:, :, 1:n + 1].transpose((1, 0, 2))       # base 2 B off 16
    check_workspace(LinAlg(), xv, np.transpose(x[:, :, 1:n + 1], (1, 0, 2)), nchan, nstand, workspace_kernels())


@pytest.mark.gpu
def test_workspace_conjugated_view():
    rng = np.random.default_rng(8)
    nstand, nchan, ntime = 12, 2, 40
    x = int_complex(rng, (nchan, ntime, 2 * nstand), 300, 'cf32')
    check_workspace(LinAlg(), bf.asarray(x, space='cuda').conj(), np.conj(x), nchan, nstand, workspace_kernels(),
                    conj=True)


@pytest.mark.gpu
def test_workspace_two_correlator_passes():
    """131076 samples: two tensor-core passes (131071 + 5), then the storage
    kernel.  Samples within +-7 keep every sum below 2^24, so the chunked sum
    is exact and equals the oracle's."""
    rng = np.random.default_rng(9)
    nstand, nchan, ntime = 8, 1, 131076
    x = np.empty((ntime, nchan, 2 * nstand), CI8)
    x['re'] = rng.integers(-7, 8, size=x.shape)
    x['im'] = rng.integers(-7, 8, size=x.shape)
    xv = bf.asarray(x, space='cuda').transpose((1, 0, 2))
    check_workspace(LinAlg(), xv, np.transpose(x, (1, 0, 2)), nchan, nstand,
                    ['corr_tc_kernel', 'corr_tc_kernel', 'vis_to_storage_kernel'])


@pytest.mark.gpu
def test_workspace_regrow():
    """One handle across a large, a small and a larger call."""
    rng = np.random.default_rng(10)
    la = LinAlg()
    for nstand, nchan, ntime in [(40, 3, 20), (9, 1, 5), (60, 4, 10)]:
        x = int_complex(rng, (nchan, ntime, 2 * nstand), 500, 'ci16')
        check_workspace(la, bf.asarray(x, space='cuda'), x, nchan, nstand, workspace_kernels())


# --------------------------------------------------------------- GPU: blocks
class ArraysSource(NumpySourceBlock):
    """One sequence per array, named seq0, seq1, ..."""

    def __init__(self, arrays, header, gulp_nframe):
        super(ArraysSource, self).__init__(arrays[0], header, gulp_nframe)
        self.arrays = arrays
        self.sourcenames = list(range(len(arrays)))

    def create_reader(self, sourcename):
        return _Reader(self.arrays[sourcename])

    def on_sequence(self, reader, sourcename):
        return [dict(self.header, name='seq%i' % sourcename)]


def run_pipeline(xs, hdr, nint, gulp, mode):
    """mode: 'two' (correlate -> convert_visibilities('storage')), 'storage'
    (correlate(output='storage')), 'fuse' (the two-block chain under
    block_scope(fuse=True)).  Returns the sequences' headers and outputs."""
    from bifrost_b200 import block_scope
    heads, outs = [], []
    with Pipeline() as p:
        src = blocks.copy(ArraysSource(xs, hdr, gulp), space='cuda')
        if mode == 'storage':
            b = blocks.correlate(src, nint, output='storage')
        else:
            with block_scope(fuse=(mode == 'fuse')):
                b = blocks.convert_visibilities(blocks.correlate(src, nint), 'storage')
        blocks.callback_sink(b, lambda s: (heads.append(s.header), outs.append([])),
                             lambda s: outs[-1].append(np.array(s.data.copy('system'))))
        p.run()
    assert (mode == 'two') == ('ConvertVisibilitiesBlock' in [type(b).__name__ for b in p.blocks])
    return heads, [np.concatenate(o, 0) for o in outs]


@pytest.mark.gpu
@pytest.mark.parametrize("nint,gulp", [(40, 40), (60, 20)])
def test_blocks_equal_the_two_block_chain(nint, gulp):
    rng = np.random.default_rng(nint + gulp)
    nchan, nstand = 3, 20
    xs = [full_range_ci8(rng, (2 * nint, nchan, nstand, 2)), full_range_ci8(rng, (nint, nchan, nstand, 2))]
    hdr = volt_header(nchan, nstand, gulp)
    got = {}
    for mode in ('two', 'storage', 'fuse'):
        kernels = []

        def run():
            got[mode] = run_pipeline(xs, hdr, nint, gulp, mode)
        kernels = ran(run)
        if mode != 'two':
            if nint == gulp:            # one fused launch per integration
                assert [k for k in kernels if 'corr' in k] == [FUSED] * 3, kernels
                assert 'vis_to_storage_kernel' not in kernels
            else:                       # three gulps summed in C, then the storage kernel
                assert kernels.count('vis_to_storage_kernel') == 3, kernels
    heads, outs = got['two']
    assert len(heads) == 2 and [o.shape[0] for o in outs] == [2, 1]
    for mode in ('storage', 'fuse'):
        assert got[mode][0] == heads
        for a, b in zip(got[mode][1], outs):
            same_bits(a, b)
    nb = nstand * (nstand + 1) // 2
    for x, out in zip(xs, outs):
        for k in range(out.shape[0]):
            xi = x[k * nint:(k + 1) * nint].reshape(nint, nchan, 2 * nstand)
            same_bits(out[k].reshape(nb, nchan, 4), oracle_storage(np.transpose(xi, (1, 0, 2)), nstand))


def closed_form_input(ntime, nchan, nstand, npol):
    """CorrelateTestInputBlock of the reference (test/test_pipeline.py:66-72)."""
    i = np.arange(nstand * npol * 2) % 255 - 127
    x = np.empty((ntime, nchan, nstand, npol), dtype=CI8)
    x['re'] = i[0::2].reshape(nstand, npol)
    x['im'] = i[1::2].reshape(nstand, npol)
    return x


@pytest.mark.gpu
def test_pipeline_correlate_to_storage_then_convert():
    """test_visibilities.py::test_pipeline_correlate_then_convert on the
    storage-output block: correlate(output='storage') -> 'matrix' equals the
    closed form, and the storage output is the oracle's Stokes of it."""
    nint, gulp, nchan, nstand, npol = 1000, 100, 128, 60, 2
    x = closed_form_input(2 * nint, nchan, nstand, npol)
    hdr = {'_tensor': {'dtype': 'ci8', 'shape': [-1, nchan, nstand, npol],
                       'labels': ['time', 'freq', 'station', 'pol'],
                       'scales': [[0, 1 / 25e3], [50e6, 25e3], None, None],
                       'units': ['s', 'Hz', None, ['X', 'Y']]},
           'name': 'corr', 'gulp_nframe': gulp}
    out = {'storage': [], 'round_trip': []}
    seqs = {}

    def sink(key, b):
        blocks.callback_sink(b, lambda s: seqs.__setitem__(key, s.header),
                             lambda s: out[key].append(np.array(s.data.copy('system'))))

    with Pipeline() as p:
        src = blocks.array_source(x, hdr, gulp_nframe=gulp)
        s = blocks.correlate(blocks.copy(src, space='cuda'), nint, output='storage')
        sink('storage', s)
        sink('round_trip', blocks.convert_visibilities(s, 'matrix'))
        p.run()
    t = seqs['round_trip']['_tensor']
    assert seqs['round_trip']['matrix_fill_mode'] == 'hermitian'
    assert seqs['round_trip']['gulp_nframe'] == seqs['storage']['gulp_nframe']
    assert t['shape'] == [-1, nchan, nstand, npol, nstand, npol] and t['dtype'] == 'cf32'
    assert t['scales'] == [[0, nint / 25e3], [50e6, 25e3], None, None, None, None]
    assert t['units'] == ['s', 'Hz', None, ['X', 'Y'], None, ['X', 'Y']]
    assert seqs['storage']['_tensor']['labels'] == ['time', 'baseline', 'freq', 'stokes']

    i = np.arange(nstand * npol * 2) % 255 - 127
    v = i[0::2] + 1j * i[1::2]
    expected = (nint * v[:, None].conj() * v[None, :]).astype(np.complex64)
    expected = np.broadcast_to(expected.reshape(nstand, npol, nstand, npol), (nchan, nstand, npol, nstand, npol))
    storage = np.concatenate(out['storage'])
    assert storage.shape[0] == 2
    for frame in storage:
        same_bits(frame, ovis.to_storage(expected))
    round_trip = np.concatenate(out['round_trip'])
    np.testing.assert_allclose(round_trip, np.broadcast_to(expected, round_trip.shape), rtol=1e-6,
                               atol=1e-6 * np.abs(expected).max())


# --------------------------------------------------------- GPU: status codes
@pytest.mark.gpu
def test_status_codes():
    h = LinAlg()

    def st(x, v):
        return _bf.bfLinAlgCorrelateToStorage(h.obj, x.as_BFarray(), v.as_BFarray())
    x = bf.zeros((3, 64, 8), 'ci8', 'cuda')
    v = bf.zeros((10, 3, 4), 'cf32', 'cuda')
    assert st(x, v) == 0
    # dtypes
    assert st(bf.zeros((3, 64, 8), 'ci4', 'cuda'), v) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    assert st(x, bf.zeros((10, 3, 4), 'cf64', 'cuda')) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    # host space
    assert st(bf.zeros((3, 64, 8), 'ci8', 'system'), v) == _bf.BF_STATUS_UNSUPPORTED_SPACE
    assert st(x, bf.zeros((10, 3, 4), 'cf32', 'system')) == _bf.BF_STATUS_UNSUPPORTED_SPACE
    # not 3-D
    assert st(bf.zeros((1, 3, 64, 8), 'ci8', 'cuda'), v) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(x, bf.zeros((1, 10, 3, 4), 'cf32', 'cuda')) == _bf.BF_STATUS_INVALID_SHAPE
    # odd n, nbaseline, channel count, nstokes
    assert st(bf.zeros((3, 64, 7), 'ci8', 'cuda'), v) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(x, bf.zeros((9, 3, 4), 'cf32', 'cuda')) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(x, bf.zeros((10, 2, 4), 'cf32', 'cuda')) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(x, bf.zeros((10, 3, 2), 'cf32', 'cuda')) == _bf.BF_STATUS_INVALID_SHAPE
    # Stokes stride
    assert st(x, bf.zeros((10, 3, 8), 'cf32', 'cuda')[..., ::2]) == _bf.BF_STATUS_UNSUPPORTED_STRIDE
    # more than 65535 channels
    assert st(bf.zeros((65536, 1, 2), 'ci8', 'cuda'), bf.zeros((1, 65536, 4), 'cf32', 'cuda')) == \
        _bf.BF_STATUS_UNSUPPORTED_SHAPE
    # x and vis overlapping
    raw = bf.zeros((3 * 64 * 8 * 2 + 10 * 3 * 4 * 8,), 'u8', 'cuda')
    xa, va = x.as_BFarray(), v.as_BFarray()
    xa.data = va.data = raw.as_BFarray().data
    assert _bf.bfLinAlgCorrelateToStorage(h.obj, xa, va) == _bf.BF_STATUS_INVALID_ARGUMENT
    bf.device.stream_synchronize()
