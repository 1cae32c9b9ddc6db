"""bfPeriodSearch*: whitened, harmonic-summed power spectra.

CPU: the oracle (oracle/period_search.py) against a per-bin loop and closed
cases, the gather identity, `significance`, the block header, Init refusals and
the exec_storage protocol on descriptor-only arrays.  GPU: bfPeriodSearchExecute
bit for bit against the oracle on batched / strided / edge-case inputs, its
statuses, workspace modes, repeatability and kernel path, and an int8
filterbank through copy -> transpose -> fdmt -> split_axis -> fft ->
period_search."""
import ctypes
import math
import os
import sys
from copy import deepcopy
from fractions import Fraction
from statistics import NormalDist

import numpy as np
import pytest

import bifrost_b200 as bf
from bifrost_b200.libbifrost import _bf, BFarray
from bifrost_b200.blocks.period_search import period_search_header, PEAK_FIELDS
from bifrost_b200.period_search import PeriodSearch, output_nblock, significance
from oracle import period_search as ops

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

LN2 = 0.6931471805599453


def noise_spec(rng, shape):
    return (rng.normal(size=shape) + 1j * rng.normal(size=shape)).astype(np.complex64)


# ------------------------------------------------------------------ oracle (CPU)
def loop_period_search(spec, nharm, window, decim):
    """The definition bin by bin in Python floats (fp64, one rounding each)."""
    nbin = spec.shape[-1]
    nlevel = nharm.bit_length()
    nblk = -(-nbin // decim)
    out = np.zeros(spec.shape[:-1] + (nlevel, nblk, 2), np.float32)
    for r in np.ndindex(*spec.shape[:-1]):
        P = [float(z.real) * float(z.real) + float(z.imag) * float(z.imag) for z in spec[r]]
        p = []
        for k in range(nbin):
            w = P[k - k % window:k - k % window + window]
            med = sorted(w)[(len(w) - 1) // 2]
            p.append(float(np.float32((P[k] / med) * LN2)) if k > 0 and med > 0 else 0.)
        S = [list(p)]
        h = 2
        while h <= nharm:
            level = []
            for k in range(nbin):
                t = 0.
                for i in range(1, h, 2):
                    t += p[math.floor(Fraction(i * k, h) + Fraction(1, 2))]   # round half up
                level.append(S[-1][k] + t)
            S.append(level)
            h *= 2
        for l, s in enumerate(S):
            for j in range(nblk):
                ks = range(j * decim, min((j + 1) * decim, nbin))
                kb = max(ks, key=lambda k: (s[k], -k))
                out[r + (l, j)] = (np.float32(s[kb]), kb - j * decim)
    return out


@pytest.mark.parametrize('nharm,window,decim,nbin', [(1, 16, 1, 40), (4, 16, 5, 77), (8, 20, 16, 100),
                                                     (32, 64, 7, 129), (16, 16, 200, 33)])
def test_oracle_equals_loop(nharm, window, decim, nbin):
    rng = np.random.default_rng(nbin)
    spec = noise_spec(rng, (2, nbin))
    spec[1, 5:9] = 0                          # ties
    got = ops.period_search(spec, nharm, window, decim)
    want = loop_period_search(spec, nharm, window, decim)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_ratio_identity():
    k = np.arange(0, (1 << 24) + 2, 997, dtype=np.int64)
    for l in range(1, 6):
        h = 1 << l
        for i in range(1, h, 2):
            q = i * 32 // h
            assert np.array_equal((2 * i * k + h) // (2 * h), (2 * q * k + 32) // 64)
    assert 2 * 31 * (1 << 24) + 32 < 2 ** 31


def test_pure_tone_lands_in_its_bin():
    n, f0 = 4096, 517
    t = np.arange(n)
    x = 10 * np.cos(2 * np.pi * f0 * t / n) + np.random.default_rng(1).normal(size=n)
    spec = np.fft.rfft(x).astype(np.complex64)[None]
    out = ops.period_search(spec, 1, 256, 64)
    j = int(np.argmax(out[0, 0, :, 0]))
    assert j * 64 + int(out[0, 0, j, 1]) == f0


def test_pulse_train_harmonics_add_up():
    n, period = 4096, 64                      # fundamental at bin n / period = 64
    x = np.random.default_rng(2).normal(size=n)
    x[::period] += 8.
    spec = np.fft.rfft(x).astype(np.complex64)[None]
    S = ops.harmonic_sums(ops.whiten(spec, 512), 32)
    fT = n // period
    at = [S[l][0, (1 << l) * fT] for l in range(6)]
    assert all(b > a for a, b in zip(at, at[1:])), at
    out = ops.peaks(S, 1)
    assert np.array_equal(out[0, :, :, 0], np.stack(S)[:, 0].astype(np.float32))


def test_zero_and_dc_only_spectra_give_zero_peaks():
    spec = np.zeros((3, 1000), np.complex64)
    spec[1, 0] = 3.7 * 1998                   # a constant series: DC only
    spec[2, 0] = -1e6
    out = ops.period_search(spec, 32, 64, 10)
    assert np.all(out == 0)


# ------------------------------------------------------------------ significance (CPU)
def test_significance_single_bin():
    S = np.array([0.01, 0.5, 1., 3., 10.])            # 1 - exp(-S) still exact enough
    want = [NormalDist().inv_cdf(1 - math.exp(-s)) for s in S]
    np.testing.assert_allclose(significance(S, 1), want, rtol=1e-9)
    assert significance(0., 8) == -np.inf
    assert np.isfinite(significance(1e4, 32)) and significance(1e4, 32) > 100


@pytest.mark.parametrize('nharm', [1, 2, 4, 8, 16, 32])
def test_significance_monotone(nharm):
    S = np.geomspace(1e-2, 1e4, 4000)
    sig = significance(S, nharm)
    assert np.all(np.isfinite(sig)) and np.all(np.diff(sig) > 0)


@pytest.mark.parametrize('nharm', [1, 2, 4, 8, 16, 32])
def test_significance_against_scipy(nharm):
    scipy_stats = pytest.importorskip('scipy.stats')
    scipy_special = pytest.importorskip('scipy.special')
    S = np.concatenate([np.geomspace(0.05, 1e4, 2000), np.linspace(0.1, 150, 2000)])
    want = -scipy_special.ndtri_exp(scipy_stats.gamma.logsf(S, nharm))
    ok = np.isfinite(want)                    # gamma.logsf underflows to -inf far out
    assert ok.sum() > 3000
    got = significance(S, nharm)
    np.testing.assert_allclose(got[ok], want[ok], rtol=1e-6, atol=1e-9)


# ------------------------------------------------------------------ header, Init (CPU)
def spectra_header(ndm=794, nfft=4096):
    """fdmt -> split_axis('time', nfft, 'fine_time') -> fft('fine_time', 'fft_freq')."""
    from bifrost_b200 import views
    from bifrost_b200.blocks.fft import FftBlock
    hdr = {'_tensor': {'dtype': 'f32', 'shape': [ndm, -1], 'labels': ['dispersion', 'time'],
                       'scales': [[0., 0.126], [12.5, 6.4e-5]], 'units': ['pc cm^-3', 's']},
           'name': 'bank', 'gulp_nframe': nfft, 'max_dm': 100.}
    t = hdr['_tensor']                        # split_axis, as views.split_axis rewrites it
    t['shape'].insert(2, nfft)
    t['units'].insert(2, 's')
    t['labels'].insert(2, 'fine_time')
    t['scales'].insert(2, [0, 6.4e-5])
    t['scales'][1] = [12.5, 6.4e-5 * nfft]
    hdr['gulp_nframe'] = 1
    t['dtype'] = 'cf32'                       # fft along fine_time
    t['shape'][2] = nfft // 2 + 1
    t['units'][2] = 'Hz'
    t['scales'][2] = [0, 1. / (6.4e-5 * nfft)]
    t['labels'][2] = 'fft_freq'
    return hdr


def test_block_header():
    ihdr = spectra_header()
    keep = deepcopy(ihdr)
    ohdr = period_search_header(ihdr, 16, 1024, 64)
    assert ihdr == keep
    t = ohdr['_tensor']
    df = 1. / (6.4e-5 * 4096)
    assert t['dtype'] == 'f32'
    assert t['shape'] == [794, -1, 5, output_nblock(2049, 64), 2]
    assert t['labels'] == ['dispersion', 'time', 'harmonic', 'fft_freq', 'peak']
    assert t['units'] == ['pc cm^-3', 's', None, 'Hz', None]
    assert t['scales'] == [[0., 0.126], [12.5, 6.4e-5 * 4096], None, [0, df * 64], None]
    assert ohdr['harmonics'] == [1, 2, 4, 8, 16]
    assert ohdr['peak_fields'] == PEAK_FIELDS == ['power', 'offset']
    assert ohdr['whiten_window'] == 1024 and ohdr['max_dm'] == 100.
    with pytest.raises(KeyError):              # frame axis last: not spectra
        period_search_header({'_tensor': dict(ihdr['_tensor'], shape=[794, 4096, -1])}, 16, 1024, 64)
    with pytest.raises(KeyError):
        period_search_header({'_tensor': dict(ihdr['_tensor'], labels=['a', 'b', 'c'])}, 16, 1024, 64)
    with pytest.raises(TypeError):
        period_search_header({'_tensor': dict(ihdr['_tensor'], dtype='f32')}, 16, 1024, 64)


def test_output_nblock():
    assert output_nblock(65537, 64) == 1025
    assert output_nblock(64, 64) == 1
    assert output_nblock(1, 1 << 24) == 1
    assert output_nblock(17, 1) == 17


@pytest.mark.parametrize('nharm,window,decim', [(0, 64, 1), (3, 64, 1), (64, 64, 1), (-1, 64, 1),
                                                (1, 15, 1), (1, 8193, 1), (1, 64, 0),
                                                (1, 64, (1 << 24) + 1)])
def test_init_rejects_bad_arguments(nharm, window, decim):
    plan = PeriodSearch()
    with pytest.raises(RuntimeError, match='INVALID_ARGUMENT'):
        plan.init(nharm, window, decim)


def test_init_accepts_limits():
    for args in ((1, 16, 1), (32, 8192, 1 << 24), (8, 100, 3)):
        PeriodSearch().init(*args)
    assert _bf.bfPeriodSearchInit(None, 1, 16, 1) == _bf.BF_STATUS_INVALID_HANDLE


# ------------------------------------------------------------------ exec_storage (CPU)
DUMMY = 1 << 32                               # 4096-aligned, never dereferenced


def desc(dtype, shape):
    a = BFarray()
    a.data = DUMMY
    a.space = _bf.BF_SPACE_CUDA
    a.dtype = {'cf32': _bf.BF_DTYPE_CF32, 'f32': _bf.BF_DTYPE_F32}[dtype]
    a.ndim = len(shape)
    stride = 8 if dtype == 'cf32' else 4
    for d in reversed(range(len(shape))):
        a.shape[d] = shape[d]
        a.strides[d] = stride
        stride *= shape[d]
    return a


def descs(nharm, decim, shape, nbin_out=None):
    nbin = shape[-1] if nbin_out is None else nbin_out
    return (desc('cf32', shape),
            desc('f32', list(shape[:-1]) + [nharm.bit_length(), output_nblock(nbin, decim), 2]))


# (nharm, window, decim, in shape, workspace bytes): p is rows x nbin f32; a
# decim above the 1024-bin tile adds (f64, i32) partials per (row, level, tile)
STORAGE = [(16, 1024, 64, [3, 4, 1000], 48128),
           (32, 16, 2000, [2, 5000], 40960),
           (1, 8192, 1, [7, 1], 256)]


@pytest.fixture(params=STORAGE, ids=['bpt', 'finish', 'tiny'])
def planned(request):
    nharm, window, decim, shape, size = request.param
    plan = ctypes.c_void_p()
    assert _bf.bfPeriodSearchCreate(ctypes.byref(plan)) == _bf.BF_STATUS_SUCCESS
    assert _bf.bfPeriodSearchInit(plan, nharm, window, decim) == _bf.BF_STATUS_SUCCESS
    x, o = descs(nharm, decim, shape)
    yield (lambda ptr, sz, h=plan: _bf.bfPeriodSearchExecute(h, ctypes.byref(x), ctypes.byref(o), ptr, sz)), size
    assert _bf.bfPeriodSearchDestroy(plan) == _bf.BF_STATUS_SUCCESS


def test_storage_query_size(planned):
    execute, size = planned
    got = _bf.BFsize(0)
    assert execute(None, ctypes.byref(got)) == _bf.BF_STATUS_SUCCESS
    assert got.value == size


def test_storage_refusals(planned):
    execute, size = planned
    short = _bf.BFsize(size - 1)
    assert execute(DUMMY, ctypes.byref(short)) == _bf.BF_STATUS_INSUFFICIENT_STORAGE
    assert execute(DUMMY, None) == _bf.BF_STATUS_INVALID_ARGUMENT


def test_handle_statuses():
    x, o = descs(4, 8, [2, 100])
    size = _bf.BFsize(0)
    assert _bf.bfPeriodSearchCreate(None) == _bf.BF_STATUS_INVALID_POINTER
    assert _bf.bfPeriodSearchDestroy(None) == _bf.BF_STATUS_INVALID_HANDLE
    assert _bf.bfPeriodSearchExecute(None, ctypes.byref(x), ctypes.byref(o), None,
                                     ctypes.byref(size)) == _bf.BF_STATUS_INVALID_HANDLE
    plan = ctypes.c_void_p()
    assert _bf.bfPeriodSearchCreate(ctypes.byref(plan)) == _bf.BF_STATUS_SUCCESS
    assert plan.value
    assert _bf.bfPeriodSearchExecute(plan, ctypes.byref(x), ctypes.byref(o), None,
                                     ctypes.byref(size)) == _bf.BF_STATUS_INVALID_STATE
    assert _bf.bfPeriodSearchDestroy(plan) == _bf.BF_STATUS_SUCCESS


@pytest.mark.parametrize('nbin', [0, (1 << 24) + 2])
def test_unsupported_bin_counts(nbin):
    plan = PeriodSearch()
    plan.init(2, 16, 64)
    x, o = descs(2, 64, [3, nbin])
    size = _bf.BFsize(0)
    assert _bf.bfPeriodSearchExecute(plan.obj, ctypes.byref(x), ctypes.byref(o), None,
                                     ctypes.byref(size)) == _bf.BF_STATUS_UNSUPPORTED_SHAPE


# ------------------------------------------------------------------ GPU
def run(d_x, nharm, window, decim, out=None):
    lead = d_x.shape[:-1]
    d_o = out if out is not None else \
        bf.zeros(lead + (nharm.bit_length(), output_nblock(d_x.shape[-1], decim), 2), 'f32', 'cuda')
    plan = PeriodSearch()
    plan.init(nharm, window, decim)
    plan.execute(d_x, d_o)
    bf.device.stream_synchronize()
    return np.asarray(d_o.copy('system'))


def same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


CASES = {
    # name: (shape, nharm, window, decim)
    'batch':            ((2, 3, 5, 3000), 16, 256, 64),
    'nbin1':            ((4, 1), 32, 16, 1),
    'nbin2':            ((4, 2), 8, 16, 3),
    'nbin17':           ((4, 17), 32, 16, 4),
    'nbin_lt_window':   ((3, 700), 8, 1024, 32),
    'nbin_eq_window':   ((3, 1024), 8, 1024, 64),
    'nbin_ragged_win':  ((3, 5000), 16, 1000, 100),
    'window16':         ((3, 2049), 32, 16, 64),
    'window8192':       ((3, 20000), 32, 8192, 64),
    'decim1':           ((3, 3001), 32, 512, 1),
    'decim_gt_nbin':    ((3, 3000), 4, 512, 5000),
    'decim_ragged':     ((3, 6001), 16, 1024, 640),
    'decim_finish':     ((3, 9000), 32, 2048, 2500),
    'decim_max':        ((2, 40000), 2, 4096, 1 << 24),
    'nharm1':           ((4, 4097), 1, 512, 64),
    'nharm32':          ((4, 65537), 32, 1024, 64),
}


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(CASES))
def test_matches_oracle(name):
    shape, nharm, window, decim = CASES[name]
    rng = np.random.default_rng(sorted(CASES).index(name))
    x = noise_spec(rng, shape)
    x.reshape(-1, shape[-1])[0, shape[-1] // 3] += 40.   # one bright bin
    got = run(bf.asarray(x, space='cuda'), nharm, window, decim)
    want = ops.period_search(x, nharm, window, decim)
    assert got.shape == want.shape
    assert same(got, want)


@pytest.mark.gpu
def test_row_pitch_and_offset_base():
    rng = np.random.default_rng(20)
    nbin, nharm, window, decim = 3000, 16, 512, 64
    big = noise_spec(rng, (2, 5, nbin + 37))
    d_big = bf.asarray(big, space='cuda')
    view = d_big[:, 1:, 1:1 + nbin]                          # ring pitch, base + one element
    nblk = output_nblock(nbin, decim)
    d_obig = bf.zeros((2, 4, 5, nblk + 3, 2), 'f32', 'cuda')
    oview = d_obig[:, :, :, 1:1 + nblk]
    plan = PeriodSearch()
    plan.init(nharm, window, decim)
    plan.execute(view, oview)
    bf.device.stream_synchronize()
    full = np.asarray(d_obig.copy('system'))
    assert same(full[:, :, :, 1:1 + nblk], ops.period_search(big[:, 1:, 1:1 + nbin], nharm, window, decim))
    assert np.all(full[:, :, :, 0] == 0) and np.all(full[:, :, :, 1 + nblk:] == 0)


@pytest.mark.gpu
def test_zero_constant_and_subnormal_rows():
    rng = np.random.default_rng(21)
    x = noise_spec(rng, (5, 4000))
    x[0] = 0
    x[1] = 0
    x[1, 0] = 3.7 * 7998                                    # constant series: DC only
    x[2] = 1.
    x[3, ::3] = 1e-20                                       # p below the f32 normal range
    got = run(bf.asarray(x, space='cuda'), 32, 256, 64)
    assert np.all(got[:2] == 0)
    assert same(got, ops.period_search(x, 32, 256, 64))


@pytest.mark.gpu
def test_nan_row_leaves_other_rows_alone():
    rng = np.random.default_rng(22)
    x = noise_spec(rng, (6, 3000))
    x[2, 1700] = np.nan
    x[4, 10] = np.inf
    got = run(bf.asarray(x, space='cuda'), 16, 512, 64)
    want = ops.period_search(x, 16, 512, 64)
    keep = [0, 1, 3, 5]
    assert same(got[keep], want[keep])


@pytest.mark.gpu
def test_config2_shape_and_repeatability():
    rng = np.random.default_rng(23)
    x = noise_spec(rng, (794, 65537))
    for r, k in ((150, 2000), (397, 31000), (700, 60000)):
        x[r, k] += 60.
    d_x = bf.asarray(x, space='cuda')
    a = run(d_x, 32, 1024, 64)
    b = run(d_x, 32, 1024, 64)
    assert a.shape == (794, 6, 1025, 2)
    assert same(a, b)
    rows = np.r_[0:16, 140:160, 390:400, 690:710, 778:794]
    assert same(a[rows], ops.period_search(x[rows], 32, 1024, 64))


@pytest.mark.gpu
def test_workspace_modes():
    rng = np.random.default_rng(24)
    for nharm, window, decim in ((16, 512, 64), (8, 256, 3000)):
        x = noise_spec(rng, (3, 4, 7000))
        d_x = bf.asarray(x, space='cuda')
        shape = (3, 4, nharm.bit_length(), output_nblock(7000, decim), 2)
        plan = PeriodSearch()
        plan.init(nharm, window, decim)
        d_a = bf.zeros(shape, 'f32', 'cuda')
        d_b = bf.zeros(shape, 'f32', 'cuda')
        size = plan.get_workspace_size(d_x, d_a)               # (NULL, &size): query only
        assert size >= 3 * 4 * 7000 * 4
        bf.device.stream_synchronize()
        assert np.all(np.asarray(d_a.copy('system')) == 0)
        plan.execute(d_x, d_a)                                  # (NULL, NULL): library-managed
        ws = bf.empty((size,), dtype='u8', space='cuda')
        plan.execute_workspace(d_x, d_b, ws.ctypes.data, size)  # (ptr, &size): caller's memory
        bf.device.stream_synchronize()
        a, b = np.asarray(d_a.copy('system')), np.asarray(d_b.copy('system'))
        assert same(a, b) and same(a, ops.period_search(x, nharm, window, decim))
        small = _bf.BFsize(size - 1)
        st = _bf.bfPeriodSearchExecute(plan.obj, d_x.as_BFarray(), d_b.as_BFarray(),
                                       ctypes.c_void_p(ws.ctypes.data), ctypes.byref(small))
        assert st == _bf.BF_STATUS_INSUFFICIENT_STORAGE
        st = _bf.bfPeriodSearchExecute(plan.obj, d_x.as_BFarray(), d_b.as_BFarray(),
                                       ctypes.c_void_p(ws.ctypes.data), None)
        assert st == _bf.BF_STATUS_INVALID_ARGUMENT


def status(plan, x, o):
    return _bf.bfPeriodSearchExecute(plan.obj, x.as_BFarray(), o.as_BFarray(), None, None)


@pytest.mark.gpu
def test_error_statuses():
    nharm, window, decim = 4, 64, 100
    plan = PeriodSearch()
    d_x = bf.zeros((2, 3, 1000), 'cf32', 'cuda')
    nblk = output_nblock(1000, decim)
    d_o = bf.zeros((2, 3, 3, nblk, 2), 'f32', 'cuda')
    assert status(plan, d_x, d_o) == _bf.BF_STATUS_INVALID_STATE
    plan.init(nharm, window, decim)
    assert status(plan, d_x, d_o) == _bf.BF_STATUS_SUCCESS
    assert status(plan, bf.zeros((2, 3, 1000), 'cf32'), d_o) == _bf.BF_STATUS_UNSUPPORTED_SPACE
    assert status(plan, d_x, bf.zeros((2, 3, 3, nblk, 2), 'f32')) == _bf.BF_STATUS_UNSUPPORTED_SPACE
    for dt in ('f32', 'cf64', 'ci16'):
        assert status(plan, bf.zeros((2, 3, 1000), dt, 'cuda'), d_o) == _bf.BF_STATUS_UNSUPPORTED_DTYPE, dt
    assert status(plan, d_x, bf.zeros((2, 3, 3, nblk, 2), 'i32', 'cuda')) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    for shape in ((3, 3, 3, nblk, 2), (2, 4, 3, nblk, 2), (2, 3, 4, nblk, 2), (2, 3, 3, nblk + 1, 2),
                  (2, 3, 3, nblk - 1, 2), (2, 3, 3, nblk, 3), (2, 3, 3, nblk)):
        assert status(plan, d_x, bf.zeros(shape, 'f32', 'cuda')) == _bf.BF_STATUS_INVALID_SHAPE, shape
    wide = bf.zeros((2, 3, 2000), 'cf32', 'cuda')
    assert status(plan, wide[:, :, ::2], d_o) == _bf.BF_STATUS_UNSUPPORTED_STRIDE
    d_o2 = bf.zeros((2, 3, 3, nblk, 4), 'f32', 'cuda')
    assert status(plan, d_x, d_o2[..., ::2]) == _bf.BF_STATUS_UNSUPPORTED_STRIDE
    huge = bf.zeros((1, (1 << 24) + 2), 'cf32', 'cuda')
    nb = output_nblock((1 << 24) + 2, decim)
    assert status(plan, huge, bf.zeros((1, 3, nb, 2), 'f32', 'cuda')) == _bf.BF_STATUS_UNSUPPORTED_SHAPE
    assert _bf.bfPeriodSearchExecute(None, d_x.as_BFarray(), d_o.as_BFarray(), None, None) == \
        _bf.BF_STATUS_INVALID_HANDLE
    assert _bf.bfPeriodSearchExecute(plan.obj, None, d_o.as_BFarray(), None, None) == \
        _bf.BF_STATUS_INVALID_POINTER
    bf.device.stream_synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize('decim,names', [(64, ('period_search_whiten_kernel', 'period_search_harmonic_kernel')),
                                         (3000, ('period_search_whiten_kernel', 'period_search_harmonic_kernel',
                                                 'period_search_finish_kernel'))])
def test_kernel_path(decim, names):
    from kernel_trace import device_kernels
    x = noise_spec(np.random.default_rng(25), (4, 8193))
    d_x = bf.asarray(x, space='cuda')
    d_o = bf.zeros((4, 6, output_nblock(8193, decim), 2), 'f32', 'cuda')
    plan = PeriodSearch()
    plan.init(32, 1024, decim)
    plan.execute(d_x, d_o)                                      # workspace allocated outside the trace
    got = device_kernels(lambda: plan.execute(d_x, d_o))
    assert len(got) == len(names)
    for g, want in zip(got, names):
        assert want in g, (got, names)


# ------------------------------------------------------------------ pipeline
@pytest.mark.gpu
def test_fdmt_fft_period_search_pipeline():
    from bifrost_b200 import blocks, views
    from bifrost_b200.pipeline import Pipeline
    nchan, md, nfft, nframe = 256, 120, 4096, 4
    ntime = nframe * nfft
    f0, df, dt = 1200., 0.5, 1e-3
    frac, period = 0.6, 61.37                                   # DM row, period in samples
    nharm, window, decim = 16, 256, 64
    rng = np.random.default_rng(26)
    x = np.clip(np.rint(rng.normal(0, 20, size=(nchan, ntime))), -127, 127).astype(np.int8)
    f = f0 + df * np.arange(nchan)
    rel = (f ** -2 - f[-1] ** -2) / (f[0] ** -2 - f[-1] ** -2)
    row = int(np.rint(frac * (md - 1)))
    for t0 in np.arange(7.0, ntime, period):
        tt = int(np.rint(t0)) + np.rint(rel * frac * (md - 1)).astype(np.int64)
        ok = tt < ntime
        x[np.arange(nchan)[ok], tt[ok]] = 40
    x = np.ascontiguousarray(x.T)
    hdr = {'_tensor': {'dtype': 'i8', 'shape': [-1, nchan], 'labels': ['time', 'freq'],
                       'scales': [[0, dt], [f0, df]], 'units': ['s', 'MHz']},
           'name': 'fil', 'gulp_nframe': nfft}
    spectra, peaks, heads = [], [], []
    with Pipeline() as p:
        src = blocks.array_source(x, hdr, gulp_nframe=nfft)
        b = blocks.copy(src, space='cuda')
        b = blocks.transpose(b, ['freq', 'time'])
        d = blocks.fdmt(b, max_delay=md)
        v = views.split_axis(d, 'time', nfft, label='fine_time')
        s = blocks.fft(v, 'fine_time', axis_labels='fft_freq')
        blocks.callback_sink(blocks.copy(s, space='system'), None,
                             lambda q: spectra.append(np.array(q.data)))
        ps = blocks.period_search(s, nharm=nharm, window=window, decim=decim)
        blocks.callback_sink(blocks.copy(ps, space='system'), lambda q: heads.append(deepcopy(q.header)),
                             lambda q: peaks.append(np.array(q.data)))
        p.run()
    spec = np.concatenate(spectra, axis=1)                      # [md, frames, nbin]
    got = np.concatenate(peaks, axis=1)                         # [md, frames, nlevel, nblk, 2]
    t = heads[0]['_tensor']
    assert t['labels'] == ['dispersion', 'time', 'harmonic', 'fft_freq', 'peak']
    assert heads[0]['harmonics'] == [1, 2, 4, 8, 16]
    assert spec.shape[1] == got.shape[1] >= 1
    for fr in range(spec.shape[1]):                            # every frame is the oracle on its spectrum
        assert same(got[:, fr], ops.period_search(np.ascontiguousarray(spec[:, fr]), nharm, window, decim))
    # the most significant peak: the injected DM row, fundamental and several harmonics
    sig = np.stack([significance(got[:, :, l, :, 0], 1 << l) for l in range(got.shape[2])], axis=2)
    r, fr, l, j = np.unravel_index(int(np.argmax(sig)), sig.shape)
    k = j * decim + int(got[r, fr, l, j, 1])
    assert abs(int(r) - row) <= 2, (r, row)
    assert abs(k / (1 << l) - nfft / period) <= 1, (k, l, nfft / period)
    assert l > 0
