"""The beamformer: bfLinAlgMatMul with cf32 / ci16 weights and ci4 / ci8
voltages (csrc/beamform.cu), ci4 on the generic kernel, the oracle and the
beamform block.

Layout of every product here, as in the reference's beamformer test:
    w [nbeam, nchan, K] -> a = w.transpose(1, 0, 2)   [nchan, nbeam, K]
    x [ntime, nchan, K] -> b = x.transpose(1, 2, 0)   [nchan, K, ntime]
    c [nchan, nbeam, ntime] (time-contiguous) or a [ntime, nchan, nbeam]
      buffer seen through .transpose(1, 2, 0) (beam-contiguous).
GPU cases assert which kernel ran (tests/kernel_trace.py)."""
import os

import numpy as np
import pytest

import bifrost_b200 as bf
from bifrost_b200.linalg import LinAlg
from bifrost_b200.pipeline import Pipeline
from oracle import beamform as obeamform
from oracle import unpack as ounpack

CI4 = bf.DataType('ci4').as_numpy_dtype()
CI8 = bf.DataType('ci8').as_numpy_dtype()
CI16 = bf.DataType('ci16').as_numpy_dtype()


def volts(rng, shape, kind):
    """Full-range voltages (-128 / -8 included) and their complex values."""
    lim = 128 if kind == 'ci8' else 8
    re = rng.integers(-lim, lim, size=shape)
    im = rng.integers(-lim, lim, size=shape)
    re.flat[0], im.flat[-1] = -lim, -lim
    if kind == 'ci8':
        x = np.empty(shape, CI8)
        x['re'], x['im'] = re, im
    else:
        x = np.empty(shape, CI4)
        x['re_im'] = ((re & 0xF) << 4 | (im & 0xF)).astype(np.uint8)
    return x, re + 1j * im


def int_weights(rng, shape, K):
    """Integer-valued cf32 weights with sum_k |w_k| |x_k| < 2^24 for |x| <= 128."""
    lim = min(127, (2 ** 24 - 1) // (2 * 128 * K))
    return (rng.integers(-lim, lim + 1, size=shape) + 1j * rng.integers(-lim, lim + 1, size=shape)).astype(np.complex64)


def kernel_name(xk, wk):
    return 'beamform_kernel<bfb::V_%s, bfb::W_%s' % (xk, wk)


def beamform_gpu(d_w, d_x, d_c, alpha=1., beta=0., reset=None):
    """Runs c = alpha a.b + beta c on the beamformer layout and returns the kernel names."""
    from kernel_trace import device_kernels
    return device_kernels(lambda: LinAlg().matmul(alpha, d_w, d_x, beta, d_c), reset=reset)


def run_case(w, x, xk, wk='cf32', c_layout='time', conj_w=False, conj_x=False):
    """Output of the new kernel (asserted) for weights w [nbeam, nchan, K] and
    voltages x [ntime, nchan, K]; returns [nchan, nbeam, ntime] complex64."""
    ntime, nchan, K = x.shape
    nbeam = w.shape[0]
    d_w = bf.asarray(w, space='cuda').transpose((1, 0, 2))
    d_x = bf.asarray(x, space='cuda').transpose((1, 2, 0))
    if conj_w:
        d_w = d_w.conj()
    if conj_x:
        d_x = d_x.conj()
    if c_layout == 'time':
        d_cbuf = bf.zeros((nchan, nbeam, ntime), 'cf32', 'cuda')
        d_c = d_cbuf
    else:
        d_cbuf = bf.zeros((ntime, nchan, nbeam), 'cf32', 'cuda')
        d_c = d_cbuf.transpose((1, 2, 0))
    names = beamform_gpu(d_w, d_x, d_c)
    assert len(names) == 1 and kernel_name(xk, wk) in names[0], names
    got = np.asarray(d_cbuf.copy('system'))
    return got if c_layout == 'time' else got.transpose(1, 2, 0)


def oracle(w, x, conj_w=False, conj_x=False):
    return obeamform.matmul_ab(w.transpose(1, 0, 2), x.transpose(1, 2, 0), conj_a=conj_w, conj_b=conj_x)


def bits(a):
    return np.ascontiguousarray(a, np.complex64).view(np.uint64)


def float_bound(w, xv):
    """sum_k |w_k| |x_k| per output [nchan, nbeam, ntime]."""
    aw = np.abs(w.astype(np.complex128)).transpose(1, 0, 2)
    ax = np.abs(xv).transpose(1, 2, 0)
    return np.matmul(aw, ax)


# ------------------------------------------------------------------ CPU: oracle
def test_oracle_against_numpy_and_reference_formula():
    rng = np.random.default_rng(1)
    a = rng.normal(size=(3, 5, 7)) + 1j * rng.normal(size=(3, 5, 7))
    b = rng.normal(size=(1, 7, 4)) + 1j * rng.normal(size=(1, 7, 4))
    want = np.matmul(a, b)
    got = obeamform.matmul_ab(a, b)
    assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()
    np.testing.assert_allclose(obeamform.matmul_ab(a, b, conj_a=True, conj_b=True),
                               np.matmul(a.conj(), b.conj()), rtol=1e-5)
    c = rng.normal(size=want.shape) + 1j * rng.normal(size=want.shape)
    np.testing.assert_allclose(obeamform.matmul_ab(a, b, 0.5, 2.0, c), 0.5 * want + 2 * c, rtol=1e-5)
    # the reference's beamformer test (test/test_linalg.py:136-151), exact integers
    ntime, nbeam, nstand, nchan = 64, 5, 32, 3
    x, xv = volts(rng, (ntime, nchan, nstand * 2), 'ci8')
    w = int_weights(rng, (nbeam, nchan, nstand * 2), nstand * 2)
    want = np.matmul(w.transpose(1, 0, 2).astype(np.complex128), xv.transpose(1, 2, 0))
    assert np.array_equal(oracle(w, x), want.astype(np.complex64))


def test_oracle_ci4_decode_against_unpack():
    """ci4 is high nibble real: bfUnpack's byte-reversed nibble order, -8 included."""
    raw = np.arange(256, dtype=np.uint8)
    x = raw.view(CI4)
    re, im, integer = obeamform._components(x, False)
    assert integer
    want = ounpack.unpack(raw.reshape(256, 1), 4, True, byte_reverse=True).reshape(256, 2)
    assert np.array_equal(re, want[:, 0]) and np.array_equal(im, want[:, 1])
    assert re[0x80] == -8 and im[0x08] == -8 and re[0x70] == 7 and im[0xFF] == -1
    assert np.array_equal(re, (raw.astype(np.int8) >> 4)) and np.array_equal(im, (raw << 4).astype(np.int8) >> 4)
    _, xv = volts(np.random.default_rng(2), (9, 4), 'ci4')
    xs, _ = volts(np.random.default_rng(2), (9, 4), 'ci4')
    re, im, _ = obeamform._components(xs, True)
    assert np.array_equal(re + 1j * im, xv.conj())


# ------------------------------------------------------------ CPU: block header
class Seq(object):
    def __init__(self, header):
        self.header = header


def volt_header(nchan=4, nstand=3, npol=2, dtype='ci8'):
    return {'_tensor': {'dtype': dtype, 'shape': [-1, nchan, nstand, npol],
                        'labels': ['time', 'freq', 'station', 'pol'],
                        'scales': [[0, 1 / 25e3], [50e6, 25e3], None, None],
                        'units': ['s', 'Hz', None, ['X', 'Y']]},
            'name': 'volts', 'gulp_nframe': 16}


def make_block(weights, dtype='ci8'):
    from bifrost_b200 import blocks
    with Pipeline():
        src = blocks.array_source(np.zeros((16, 4, 3, 2), CI8), volt_header(), gulp_nframe=16)
        return blocks.beamform(src, weights)


def test_block_header_contract():
    w = np.ones((4, 5, 3, 2), np.complex64)
    ohdr = make_block(w).on_sequence(Seq(volt_header()))
    t = ohdr['_tensor']
    assert t['labels'] == ['time', 'freq', 'beam'] and t['dtype'] == 'cf32'
    assert t['shape'] == [-1, 4, 5]
    assert t['scales'] == [[0, 1 / 25e3], [50e6, 25e3], None]
    assert t['units'] == ['s', 'Hz', None]
    assert ohdr['name'] == 'volts' and ohdr['gulp_nframe'] == 16
    for dtype in ('ci4', 'ci16', 'cf32'):
        assert make_block(w).on_sequence(Seq(volt_header(dtype=dtype)))['_tensor']['dtype'] == 'cf32'


def test_block_rejects_bad_input():
    w = np.ones((4, 5, 3, 2), np.complex64)
    bad = volt_header()
    bad['_tensor']['labels'] = ['time', 'freq', 'pol', 'station']
    with pytest.raises(ValueError):
        make_block(w).on_sequence(Seq(bad))
    with pytest.raises(ValueError):
        make_block(w).on_sequence(Seq(volt_header(dtype='i8')))
    for shape in [(3, 5, 3, 2), (4, 5, 2, 2), (4, 5, 3, 1)]:
        with pytest.raises(ValueError):
            make_block(np.ones(shape, np.complex64)).on_sequence(Seq(volt_header()))
    with pytest.raises(ValueError):
        make_block(np.ones((4, 5, 3, 2), np.float32))


def test_kernels_compile_without_spills(tmp_path):
    """The beamformer's sm_90a build: every instantiation, no local-memory spills."""
    import subprocess
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'bifrost_b200', 'csrc')
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    out = subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17',
                          '-I' + os.path.join(src, '..', '..', 'include'), '-I' + src, '--expt-relaxed-constexpr',
                          '-Xptxas', '-v', '-c', os.path.join(src, 'beamform.cu'), '-o', str(tmp_path / 'b.o')],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    entries = [l for l in out.stderr.splitlines() if 'Compiling entry function' in l and 'beamform_kernel' in l]
    assert len(entries) == 20
    spills = [l for l in out.stderr.splitlines() if 'spill stores' in l]
    assert spills and all(' 0 bytes spill stores, 0 bytes spill loads' in l for l in spills), spills


# -------------------------------------------------------------- GPU: exactness
NBEAMS = list(range(1, 18)) + [64, 100]
KS = [1, 2, 3, 34, 512, 704]
NTIMES = [1, 7, 64, 513, 4096]
NCHANS = [1, 3, 10]


def exact_case(nbeam, K, ntime, nchan, xk, seed):
    if ntime * nchan * K > 4096 * 10 * 128:          # keep each case's host oracle small
        nchan = 1
    rng = np.random.default_rng(seed)
    x, xv = volts(rng, (ntime, nchan, K), xk)
    w = int_weights(rng, (nbeam, nchan, K), K)
    got = run_case(w, x, xk)
    assert np.array_equal(bits(got), bits(oracle(w, x)))


@pytest.mark.gpu
@pytest.mark.parametrize("xk", ['ci8', 'ci4'])
@pytest.mark.parametrize("i,nbeam", list(enumerate(NBEAMS)))
def test_exact_sweep_nbeam(i, nbeam, xk):
    exact_case(nbeam, KS[i % len(KS)], NTIMES[(i // 2) % len(NTIMES)], NCHANS[i % len(NCHANS)], xk, 100 + i)


@pytest.mark.gpu
@pytest.mark.parametrize("xk", ['ci8', 'ci4'])
@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("j,ntime", list(enumerate(NTIMES)))
def test_exact_sweep_k_ntime(j, ntime, K, xk):
    nbeam = NBEAMS[(j * 7 + KS.index(K)) % len(NBEAMS)]
    exact_case(nbeam, K, ntime, NCHANS[(j + KS.index(K)) % len(NCHANS)], xk, 1000 + 10 * j + K)


# ---------------------------------------------------------- GPU: float weights
@pytest.mark.gpu
@pytest.mark.parametrize("xk", ['ci8', 'ci4'])
@pytest.mark.parametrize("wk", ['cf32', 'ci16'])
@pytest.mark.parametrize("nbeam,K,ntime,nchan", [(1, 512, 4096, 2), (5, 34, 513, 3), (16, 703, 300, 2), (37, 256, 257, 1)])
def test_float_weights(nbeam, K, ntime, nchan, wk, xk):
    rng = np.random.default_rng(nbeam * K + ntime)
    x, xv = volts(rng, (ntime, nchan, K), xk)
    if wk == 'cf32':
        w = (rng.normal(size=(nbeam, nchan, K)) + 1j * rng.normal(size=(nbeam, nchan, K))).astype(np.complex64)
        wv = w
    else:
        w = np.empty((nbeam, nchan, K), CI16)
        w['re'] = rng.choice([-32767, 32767, -32768, 1, 0], size=w.shape)
        w['im'] = rng.integers(-32768, 32768, size=w.shape)
        wv = w['re'] + 1j * w['im'].astype(np.float64)
    got = run_case(w, x, xk, wk)
    want = np.matmul(wv.astype(np.complex128).transpose(1, 0, 2), xv.transpose(1, 2, 0))
    err = np.maximum(np.abs(got.real - want.real), np.abs(got.imag - want.imag))
    assert np.all(err <= 1e-6 * float_bound(wv, xv)), err.max()
    if wk == 'cf32':
        # the same call on the generic kernel agrees within the same bound
        os.environ['BFB_LINALG_SIMT'] = '1'
        try:
            d_c = bf.zeros((nchan, nbeam, ntime), 'cf32', 'cuda')
            names = beamform_gpu(bf.asarray(w, space='cuda').transpose((1, 0, 2)),
                                 bf.asarray(x, space='cuda').transpose((1, 2, 0)), d_c)
        finally:
            del os.environ['BFB_LINALG_SIMT']
        assert len(names) == 1 and 'matmul_ab_kernel<float>' in names[0], names
        simt = np.asarray(d_c.copy('system'))
        err = np.maximum(np.abs(got.real - simt.real), np.abs(got.imag - simt.imag))
        assert np.all(err <= 2e-6 * float_bound(wv, xv)), err.max()


# -------------------------------------------------------------- GPU: invariants
@pytest.mark.gpu
def test_ci4_equals_unpacked_ci8():
    """ci4 in, and the same data through bfUnpack (byte-reversed nibble order:
    high nibble real) to ci8, give the same bits."""
    rng = np.random.default_rng(5)
    ntime, nchan, K, nbeam = 1000, 3, 130, 6
    x4, _ = volts(rng, (ntime, nchan, K), 'ci4')
    w = (rng.normal(size=(nbeam, nchan, K)) + 1j * rng.normal(size=(nbeam, nchan, K))).astype(np.complex64)
    d4 = bf.asarray(bf.ndarray(x4, dtype='ci4'), space='cuda')
    d8 = bf.empty((ntime, nchan, K), 'ci8', 'cuda')
    bf.unpack(bf.asarray(bf.ndarray(x4, dtype="ci4").byteswap(), space="cuda"), d8)
    x8 = np.asarray(d8.copy('system'))
    assert np.array_equal(x8['re'], x4['re_im'].astype(np.int8) >> 4)
    out = []
    for d, xk in ((d4, 'ci4'), (d8, 'ci8')):
        d_c = bf.zeros((nchan, nbeam, ntime), 'cf32', 'cuda')
        names = beamform_gpu(bf.asarray(w, space='cuda').transpose((1, 0, 2)), d.transpose((1, 2, 0)), d_c)
        assert kernel_name(xk, 'cf32') in names[0]
        out.append(np.asarray(d_c.copy('system')))
    assert np.array_equal(bits(out[0]), bits(out[1]))


@pytest.mark.gpu
@pytest.mark.parametrize("xk", ['ci8', 'ci4'])
def test_misaligned_base_layouts_and_repeat(xk):
    """A [..., 1:] slice (any byte phase), time- and beam-contiguous C, and
    two identical calls: all bitwise equal."""
    rng = np.random.default_rng(6)
    ntime, nchan, K, nbeam = 700, 3, 77, 9
    xbig, xvbig = volts(rng, (ntime, nchan, K + 1), xk)
    w = (rng.normal(size=(nbeam, nchan, K)) + 1j * rng.normal(size=(nbeam, nchan, K))).astype(np.complex64)
    d_big = bf.asarray(xbig, space='cuda')
    x_al = np.ascontiguousarray(xbig[..., 1:])
    ref = run_case(w, x_al, xk)
    ref2 = run_case(w, x_al, xk)
    beam = run_case(w, x_al, xk, c_layout='beam')
    assert np.array_equal(bits(ref), bits(ref2)) and np.array_equal(bits(ref), bits(beam))
    d_c = bf.zeros((nchan, nbeam, ntime), 'cf32', 'cuda')
    names = beamform_gpu(bf.asarray(w, space='cuda').transpose((1, 0, 2)), d_big[..., 1:].transpose((1, 2, 0)), d_c)
    assert kernel_name(xk, 'cf32') in names[0]
    assert np.array_equal(bits(np.asarray(d_c.copy('system'))), bits(ref))
    # padded K row stride: stations sliced out of a wider array
    d_c = bf.zeros((nchan, nbeam, ntime), 'cf32', 'cuda')
    names = beamform_gpu(bf.asarray(w, space='cuda').transpose((1, 0, 2)), d_big[..., :K].transpose((1, 2, 0)), d_c)
    assert kernel_name(xk, 'cf32') in names[0]
    want = run_case(w, np.ascontiguousarray(xbig[..., :K]), xk)
    assert np.array_equal(bits(np.asarray(d_c.copy('system'))), bits(want))


# --------------------------------------------------------- GPU: views, operands
@pytest.mark.gpu
@pytest.mark.parametrize("xk", ['ci8', 'ci4'])
@pytest.mark.parametrize("conj_w,conj_x", [(True, False), (False, True), (True, True)])
def test_conjugated_views(conj_w, conj_x, xk):
    rng = np.random.default_rng(7)
    x, _ = volts(rng, (300, 2, 40), xk)
    w = int_weights(rng, (5, 2, 40), 40)
    got = run_case(w, x, xk, conj_w=conj_w, conj_x=conj_x)
    assert np.array_equal(bits(got), bits(oracle(w, x, conj_w, conj_x)))


@pytest.mark.gpu
@pytest.mark.parametrize("c_layout", ['time', 'beam'])
def test_alpha_beta_nan_and_padding(c_layout):
    """alpha / beta; beta = 0 never reads C (NaN there must not show); a
    sentinel in C's padding survives."""
    rng = np.random.default_rng(8)
    ntime, nchan, K, nbeam = 300, 2, 64, 6
    x, _ = volts(rng, (ntime, nchan, K), 'ci8')
    w = int_weights(rng, (nbeam, nchan, K), K)
    d_w = bf.asarray(w, space='cuda').transpose((1, 0, 2))
    d_x = bf.asarray(x, space='cuda').transpose((1, 2, 0))
    sentinel = np.complex64(-12345 + 678j)
    if c_layout == 'time':
        buf = np.full((nchan, nbeam + 1, ntime + 3), sentinel, np.complex64)
        buf[:, :nbeam, :ntime] = np.nan
        d_buf = bf.asarray(buf, space='cuda')
        d_c = d_buf[:, :nbeam, :ntime]
        view = lambda a: a[:, :nbeam, :ntime]             # noqa: E731
    else:
        buf = np.full((ntime, nchan, nbeam + 2), sentinel, np.complex64)
        buf[:, :, :nbeam] = np.nan
        d_buf = bf.asarray(buf, space='cuda')
        d_c = d_buf[:, :, :nbeam].transpose((1, 2, 0))
        view = lambda a: a[:, :, :nbeam].transpose(1, 2, 0)   # noqa: E731
    names = beamform_gpu(d_w, d_x, d_c, alpha=0.5, beta=0.)
    assert kernel_name('ci8', 'cf32') in names[0]
    got = np.asarray(d_buf.copy('system'))
    want = obeamform.matmul_ab(w.transpose(1, 0, 2), x.transpose(1, 2, 0), alpha=0.5)
    assert np.array_equal(bits(view(got)), bits(want))
    pad = np.ones(got.shape, bool)
    if c_layout == 'time':
        pad[:, :nbeam, :ntime] = False
    else:
        pad[:, :, :nbeam] = False
    assert np.all(got[pad] == sentinel)
    names = beamform_gpu(d_w, d_x, d_c, alpha=2., beta=-1.5)
    assert kernel_name('ci8', 'cf32') in names[0]
    want2 = obeamform.matmul_ab(w.transpose(1, 0, 2), x.transpose(1, 2, 0), alpha=2., beta=-1.5, c=want)
    got2 = np.asarray(d_buf.copy('system'))
    assert np.array_equal(bits(view(got2)), bits(want2))
    assert np.all(got2[pad] == sentinel)


@pytest.mark.gpu
@pytest.mark.parametrize("xk", ['ci8', 'ci4'])
def test_broadcast_weights(xk):
    """One weight set [1, nbeam, K] for every channel."""
    rng = np.random.default_rng(9)
    ntime, nchan, K, nbeam = 260, 5, 48, 3
    x, _ = volts(rng, (ntime, nchan, K), xk)
    w1 = int_weights(rng, (1, nbeam, K), K)
    d_c = bf.zeros((nchan, nbeam, ntime), 'cf32', 'cuda')
    names = beamform_gpu(bf.asarray(w1, space='cuda'), bf.asarray(x, space='cuda').transpose((1, 2, 0)), d_c)
    assert len(names) == 1 and kernel_name(xk, 'cf32') in names[0]
    want = obeamform.matmul_ab(w1, x.transpose(1, 2, 0))
    assert np.array_equal(bits(np.asarray(d_c.copy('system'))), bits(want))


@pytest.mark.gpu
@pytest.mark.parametrize("operand", ['a', 'b'])
def test_ci4_on_the_generic_kernel(operand):
    """ci4 as either operand, in layouts the beamformer does not take (ci4
    weights; ci4 voltages with K not unit stride)."""
    rng = np.random.default_rng(10)
    m, k, n = 13, 21, 17
    if operand == 'a':
        a, _ = volts(rng, (m, k), 'ci4')
        b = (rng.integers(-9, 10, size=(k, n)) + 1j * rng.integers(-9, 10, size=(k, n))).astype(np.complex64)
    else:
        a = (rng.integers(-9, 10, size=(m, k)) + 1j * rng.integers(-9, 10, size=(m, k))).astype(np.complex64)
        b, _ = volts(rng, (k, n), 'ci4')
    d_c = bf.zeros((m, n), 'cf32', 'cuda')
    names = beamform_gpu(bf.asarray(a, space='cuda'), bf.asarray(b, space='cuda'), d_c)
    assert len(names) == 1 and 'matmul_ab_kernel<float>' in names[0], names
    assert np.array_equal(bits(np.asarray(d_c.copy('system'))), bits(obeamform.matmul_ab(a, b)))


# -------------------------------------------------------------- GPU: pipeline
@pytest.mark.gpu
@pytest.mark.parametrize("xk", ['ci8', 'ci4'])
def test_pipeline_two_sequences(xk):
    """beamform in a ring pipeline: a gulp that does not divide the sequence,
    two sequences with their own weights check, output bit-equal to the oracle."""
    from bifrost_b200 import blocks
    rng = np.random.default_rng(11)
    ntime, nchan, nstand, npol, nbeam, gulp = 700, 3, 12, 2, 4, 256
    x, _ = volts(rng, (ntime, nchan, nstand, npol), xk)
    w = int_weights(rng, (nchan, nbeam, nstand, npol), nstand * npol)
    hdr = volt_header(nchan, nstand, npol, xk)
    hdr['gulp_nframe'] = gulp
    outs, seqs = ([], []), []

    def sink(b, i):
        blocks.callback_sink(b, lambda s: seqs.append(s.header),
                             lambda s: outs[i].append(np.array(s.data.copy('system'))))

    src_x = (lambda a: bf.ndarray(a, dtype='ci4')) if xk == 'ci4' else (lambda a: a)
    with Pipeline() as p:
        # two sequences of different lengths through two beamformers
        for i, n in enumerate((ntime, 300)):
            src = blocks.array_source(src_x(x[:n]), hdr, gulp_nframe=gulp)
            sink(blocks.beamform(blocks.copy(src, space='cuda'), w), i)
        p.run()
    assert len(seqs) == 2
    for s in seqs:
        t = s['_tensor']
        assert t['shape'] == [-1, nchan, nbeam] and t['labels'] == ['time', 'freq', 'beam']
    wk = w.reshape(nchan, nbeam, nstand * npol)
    xf = x.reshape(ntime, nchan, nstand * npol)
    for i, n in enumerate((ntime, 300)):
        got = np.concatenate(outs[i], 0)
        want = obeamform.matmul_ab(wk, xf[:n].transpose(1, 2, 0)).transpose(2, 0, 1)
        assert got.shape == (n, nchan, nbeam)
        assert np.array_equal(bits(got), bits(want))


# ---------------------------------------------------------- reference golden
def _golden():
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from golden import make_ref_beamform_golden as refgold
    return refgold, refgold.load()


def test_oracle_matches_the_reference_golden():
    """The reference's own bfLinAlgMatMul (bf_cgemm_TN_smallM) gave the stored
    samples (tests/golden/make_ref_beamform_golden.py) over the shapes of its
    beamformer test; the oracle reproduces every one bit for bit, ci4 included,
    so the reference decodes ci4 as high nibble real too."""
    refgold, gold = _golden()
    assert len(gold.files) == len(refgold.CASES) == 162
    for ci in range(len(refgold.CASES)):
        x, w = refgold.case_inputs(ci)
        want = oracle(w, x).ravel()
        assert np.array_equal(bits(want[refgold.sample_index(want.size, ci)]), bits(gold[refgold.key(ci)])), \
            refgold.key(ci)


@pytest.mark.gpu
@pytest.mark.parametrize("xk", ['ci4', 'ci8'])
def test_matches_the_reference_golden(xk):
    """Our kernel against the reference's stored outputs, bit for bit."""
    refgold, gold = _golden()
    for ci, case in enumerate(refgold.CASES):
        if case[0] != xk:
            continue
        x, w = refgold.case_inputs(ci)
        got = run_case(w, x, xk).ravel()
        assert np.array_equal(bits(got[refgold.sample_index(got.size, ci)]), bits(gold[refgold.key(ci)])), \
            refgold.key(ci)
