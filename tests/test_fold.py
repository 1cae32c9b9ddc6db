"""bfFold*: phase-binned pulsar profiles.

CPU: the oracle (oracle/fold.py) against a per-sample loop, phase 0 at
tau = 0, the bin edge below one turn, negative tau, nbin = 1, split
invariance of the bins, dispersion_delays, the block header and Init's
argument checks.  GPU: bfFoldExecute against the oracle for u8 / u16 / f32
(batched, strided, offset-by-one, negative df, nbin 1 ... 4096, slow and fast
spins, spin-down terms, t0 of +-1e5 s, non-finite rows), one call against
accumulated calls over an uneven split, repeatability, the workspace
protocol, every status code and the kernel path; and two pipelines: a GUPPI
RAW pulse train through read_guppi_raw -> copy -> transpose -> merge_axes ->
coherent_dedisp -> detect -> fold, and a u8 filterbank through transpose ->
fold."""
import ctypes
import math
import os
import sys
from copy import deepcopy

import numpy as np
import pytest

import bifrost_b200 as bf
from bifrost_b200.libbifrost import _bf
from bifrost_b200.fold import Fold, dispersion_delays
from bifrost_b200.coherent_dedisp import KDM, dispersion_overlap, default_nfft
from bifrost_b200.blocks.fold import fold_header
from oracle import fold as ofold

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------ oracle (CPU)
def loop_bin(a, t, tsamp, nu, nudot, nuddot, nbin):
    tau = a + float(t) * tsamp
    c2, c3 = 0.5 * nudot, nuddot / 6.0
    phi = ((c3 * tau + c2) * tau + nu) * tau
    frac = phi - math.floor(phi)
    return min(int(math.floor(frac * nbin)), nbin - 1)


def test_oracle_matches_per_sample_loop():
    rng = np.random.default_rng(0)
    nchan, nbat, ntime, nbin = 3, 2, 700, 37
    delays = [0.0, 1.3e-3, 2.9e-2]
    tsamp, t0, nu, nudot, nuddot, first = 1e-4, -12.5, 13.7, -2e-3, 1e-6, 12345
    x = rng.normal(size=(nchan, nbat, ntime)).astype(np.float32)
    sums, counts = ofold.fold(x, nbin, delays, tsamp, t0, nu, nudot, nuddot, first)
    want_s = np.zeros((nchan, nbat, nbin))
    want_n = np.zeros((nchan, nbin), np.int64)
    for c in range(nchan):
        a = t0 - delays[c]
        for t in range(ntime):
            b = loop_bin(a, first + t, tsamp, nu, nudot, nuddot, nbin)
            want_n[c, b] += 1
            for r in range(nbat):
                want_s[c, r, b] += float(x[c, r, t])
    assert np.array_equal(counts, want_n)
    assert np.abs(sums - want_s).max() < 1e-9


def test_phase_zero_at_tau_zero():
    b = ofold.bins(1, 4, 64, [0.0], 0.25, 0.0, 1.0)
    assert list(b[0]) == [0, 16, 32, 48]
    b = ofold.bins(2, 3, 10, [0.0, 0.5], 0.5, 0.5, 1.0)      # channel 1: tau = 0 at sample 0
    assert list(b[1]) == [0, 5, 0] and list(b[0]) == [5, 0, 5]


def test_frac_just_below_one_goes_to_last_bin():
    # phi = -1e-20: floor -1, frac = 1 - 1e-20 rounds to 1.0, floor(nbin) = nbin -> nbin - 1
    assert ofold.bins(1, 1, 8, [0.0], 1.0, -1e-20, 1.0)[0, 0] == 7
    # frac = 1 - 2^-40 stays below one and is in the last bin too
    assert ofold.bins(1, 1, 4096, [0.0], 1.0, 1.0 - 2.0 ** -40, 1.0)[0, 0] == 4095
    assert ofold.bins(1, 1, 8, [0.0], 1.0, 0.875, 1.0)[0, 0] == 7
    assert ofold.bins(1, 1, 8, [0.0], 1.0, 0.875 - 1e-12, 1.0)[0, 0] == 6


def test_negative_tau():
    b = ofold.bins(1, 3, 10, [0.0], 1.0, -10.25, 1.0)        # phases -10.25, -9.25, -8.25
    assert list(b[0]) == [7, 7, 7]
    b = ofold.bins(1, 1, 10, [0.0], 1.0, -0.05, 2.0)          # phi = -0.1: frac 0.9
    assert b[0, 0] == 9


def test_nbin_one():
    rng = np.random.default_rng(1)
    x = rng.integers(0, 256, size=(2, 500)).astype(np.uint8)
    sums, counts = ofold.fold(x, 1, [0.0, 1e-3], 1e-3, 3.3, 17.0)
    assert np.array_equal(counts, [[500], [500]])
    assert np.array_equal(sums[:, 0], x.sum(axis=1))


@pytest.mark.parametrize('first', [0, 1, 999, 123456789, 1 << 40])
def test_bins_split_invariance(first):
    """Calls on [first, first + 2000) and on any split of it bin every sample
    alike: time enters only through the integer first + t."""
    args = (2, [0.0, 0.0123], 6.4e-7, 1e5, 641.9, -1e-10, 1e-20)
    part = ofold.bins(args[0], 2000, 1024, *args[1:], first=first)
    if first <= 10000:
        whole = ofold.bins(args[0], first + 2000, 1024, *args[1:])
        assert np.array_equal(whole[:, first:], part)
    for a, b in ((0, 1), (1, 700), (700, 2000)):
        piece = ofold.bins(args[0], b - a, 1024, *args[1:], first=first + a)
        assert np.array_equal(piece, part[:, a:b])


def test_dispersion_delays():
    d = dispersion_delays([1000.0, 1500.0, 2000.0], 10.0, 2000.0)
    assert abs(d[0] - 4.148741601e3 * 10 * (1e-6 - 0.25e-6)) < 1e-15
    assert abs(d[1] - 4.148741601e3 * 10 * (1 / 1500.0 ** 2 - 0.25e-6)) < 1e-15
    assert d[2] == 0.0
    # 4148.741601 x 56.7 x (1/400^2 - 1/800^2) = 4148.741601 x 56.7 x 4.6875e-6
    assert abs(dispersion_delays([400.0], 56.7, 800.0)[0] - 1.10265772864) < 1e-10
    assert dispersion_delays([1400.0], 0.0, 1500.0)[0] == 0.0
    assert KDM == 4.148741601e3


def filterbank_header(nchan=8, f0=1400.0, df=-0.5, tsamp=64e-6, dtype='u8', gulp=4096, origin=1.6e9,
                      labels=('freq', 'time')):
    shape = [nchan, -1] if len(labels) == 2 else [nchan, 4, -1]
    scales = [[f0, df], [origin, tsamp]] if len(labels) == 2 else [[f0, df], None, [origin, tsamp]]
    units = ['MHz', 's'] if len(labels) == 2 else ['MHz', None, 's']
    return {'_tensor': {'dtype': dtype, 'shape': shape, 'labels': list(labels), 'scales': scales, 'units': units},
            'name': 'fil', 'gulp_nframe': gulp}


def test_block_header_plain_reversed_band():
    ihdr = filterbank_header()
    keep = deepcopy(ihdr)
    ohdr, delays, tsamp, t0, nsub = fold_header(ihdr, 256, 1.4, dm=56.0)
    assert ihdr == keep
    t = ohdr['_tensor']
    assert t['dtype'] == 'f32' and t['shape'] == [-1, 8, 256] and t['labels'] == ['time', 'freq', 'phase']
    assert t['scales'] == [[1.6e9, 64e-6 * 4096], [1400.0, -0.5], [0.0, 1.0 / 256]]
    assert t['units'] == ['s', 'MHz', None]
    assert ohdr['gulp_nframe'] == 1 and nsub == 4096 and tsamp == 64e-6 and t0 == 0.0
    # reversed band: channel 0 is the highest centre and the reference
    freqs = 1400.0 - 0.5 * np.arange(8)
    assert ohdr['fold_fref'] == 1400.0 and delays[0] == 0.0 and np.all(delays[1:] > 0)
    assert np.array_equal(delays, dispersion_delays(freqs, 56.0, 1400.0))
    assert ohdr['fold_nbin'] == 256 and ohdr['fold_nu'] == 1.4 and ohdr['fold_nudot'] == 0.0
    assert ohdr['fold_nuddot'] == 0.0 and ohdr['fold_pepoch'] is None and ohdr['fold_dm'] == 56.0
    assert ohdr['fold_nsamp_sub'] == 4096
    # a negative time step (reversed GUPPI band) folds at |step|
    neg = filterbank_header(tsamp=-64e-6)
    assert fold_header(neg, 16, 1.4, dm=1.0)[2] == 64e-6
    assert fold_header(neg, 16, 1.4, dm=1.0)[0]['_tensor']['scales'][0] == [1.6e9, 64e-6 * 4096]
    # pepoch: t0 = origin - (pepoch - 40587) 86400
    _, _, _, t0, _ = fold_header(ihdr, 16, 1.4, pepoch=58849.5, dm=1.0)
    assert t0 == 1.6e9 - (58849.5 - 40587) * 86400.0
    assert fold_header(ihdr, 16, 1.4, pepoch=58849.5, dm=1.0)[0]['fold_pepoch'] == 58849.5


def test_block_header_coherent():
    ihdr = filterbank_header(nchan=4, f0=400.78125, df=1.5625, tsamp=0.64e-6, dtype='f32',
                             labels=('freq', 'pol', 'time'))
    ihdr.update(coherent_dm=12.0, coherent_dm_units='pc cm^-3')
    ohdr, delays, tsamp, t0, nsub = fold_header(ihdr, 64, 100.0, 1e-3, 2e-6, tsubint=4096 * 3 * 0.64e-6)
    tops = 400.78125 + 1.5625 * np.arange(4) + 0.78125
    assert ohdr['fold_fref'] == tops[-1] and ohdr['fold_dm'] == 12.0 and nsub == 3 * 4096
    assert np.array_equal(delays, dispersion_delays(tops, 12.0, tops[-1]))
    t = ohdr['_tensor']
    assert t['shape'] == [-1, 4, 4, 64] and t['labels'] == ['time', 'freq', 'pol', 'phase']
    assert t['scales'][1] == [400.78125, 1.5625] and t['scales'][2] is None
    assert t['units'] == ['s', 'MHz', None, None]
    assert ohdr['fold_nudot'] == 1e-3 and ohdr['fold_nuddot'] == 2e-6
    assert abs(t['scales'][0][1] - 3 * 4096 * 0.64e-6) < 1e-18
    # an explicit dm overrides coherent_dm
    assert fold_header(ihdr, 64, 100.0, dm=3.0)[0]['fold_dm'] == 3.0


def test_block_header_rejects():
    ihdr = filterbank_header()
    with pytest.raises(ValueError):                 # no dm and no coherent_dm
        fold_header(ihdr, 16, 1.4)
    for tsub in (4095 * 64e-6, 0.0, 6000 * 64e-6, -4096 * 64e-6):
        with pytest.raises(ValueError):
            fold_header(ihdr, 16, 1.4, dm=1.0, tsubint=tsub)
    assert fold_header(ihdr, 16, 1.4, dm=1.0, tsubint=8192 * 64e-6)[4] == 8192
    with pytest.raises(ValueError):                 # 2^31 samples would wrap a count
        fold_header(ihdr, 16, 1.4, dm=1.0, tsubint=(1 << 31) * 64e-6)
    assert fold_header(ihdr, 16, 1.4, dm=1.0, tsubint=((1 << 31) - 4096) * 64e-6)[4] == (1 << 31) - 4096
    for dt in ('i8', 'cf32', 'ci8', 'f64'):
        with pytest.raises(TypeError):
            fold_header(filterbank_header(dtype=dt), 16, 1.4, dm=1.0)
    with pytest.raises(KeyError):
        fold_header(filterbank_header(labels=('time', 'freq')), 16, 1.4, dm=1.0)
    bad = filterbank_header()
    bad['_tensor']['shape'] = [-1, 4096]
    with pytest.raises(KeyError):
        fold_header(bad, 16, 1.4, dm=1.0)


def init_status(nbin=64, delays=(0.0, 1e-3), tsamp=1e-3, t0=0.0, nu=1.0, nudot=0.0, nuddot=0.0):
    p = Fold()
    if delays is None:
        ptr, n = None, 2
    else:
        d = np.asarray(delays, np.float64)
        ptr, n = d.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), d.size
    return _bf.bfFoldInit(p.obj, nbin, n, ptr, tsamp, t0, nu, nudot, nuddot)


@pytest.mark.parametrize('kw', [
    dict(nbin=0), dict(nbin=4097), dict(nbin=-1),
    dict(tsamp=0.0), dict(tsamp=-1e-3), dict(tsamp=float('nan')), dict(tsamp=float('inf')),
    dict(nu=0.0), dict(nu=-1.0), dict(nu=float('nan')), dict(nu=float('inf')),
    dict(t0=float('nan')), dict(t0=float('-inf')),
    dict(nudot=float('nan')), dict(nudot=float('inf')), dict(nuddot=float('nan')), dict(nuddot=float('-inf')),
    dict(delays=(0.0, float('nan'))), dict(delays=(float('inf'), 0.0)), dict(delays=()),
])
def test_init_rejects_bad_arguments(kw):
    assert init_status(**kw) == _bf.BF_STATUS_INVALID_ARGUMENT


def test_init_checks_pointer_handle_and_limits():
    assert init_status(delays=None) == _bf.BF_STATUS_INVALID_POINTER
    d = np.zeros(1)
    assert _bf.bfFoldInit(None, 8, 1, d.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), 1e-3, 0., 1., 0., 0.) \
        == _bf.BF_STATUS_INVALID_HANDLE
    for nbin in (1, 7, 4096):
        assert init_status(nbin=nbin) == _bf.BF_STATUS_SUCCESS
    assert init_status(t0=-1e5, nudot=-1e-10, nuddot=1e-20) == _bf.BF_STATUS_SUCCESS
    p = Fold()
    p.init(16, [0.0, 0.1, 0.2], 1e-3, 5.0, 2.0)
    assert p.nchan == 3 and p.nbin == 16


# ------------------------------------------------------------------ GPU
def host(d):
    return np.asarray(d.copy('system'))


def make_input(rng, dtype, shape):
    if dtype == 'u8':
        return rng.integers(0, 256, size=shape).astype(np.uint8)
    if dtype == 'u16':
        return rng.integers(0, 65536, size=shape).astype(np.uint16)
    return (rng.normal(size=shape) * 10 + 3).astype(np.float32)


def check_sums(got, want, x, dtype):
    """u8 / u16: bit for bit; f32: within one f32 ulp of the fp64 oracle (plus
    the fp64 rounding of the two summation orders, 1e-12 of the bin's sum of
    magnitudes, for bins that cancel to near zero)."""
    want32 = want.astype(np.float32)
    if dtype != 'f32':
        assert np.array_equal(got.view(np.uint32), want32.view(np.uint32))
        return
    fin = np.isfinite(want)
    assert np.array_equal(np.isnan(got), np.isnan(want)), "NaN bins differ"
    assert np.array_equal(got[~fin & ~np.isnan(want)], want32[~fin & ~np.isnan(want)])
    err = np.abs(got[fin].astype(np.float64) - want[fin])
    tol = np.spacing(np.abs(want32[fin])).astype(np.float64) + 1e-12 * np.abs(x).sum() / max(1, want.size)
    assert np.all(err <= tol), (err.max(), tol[np.argmax(err - tol)])


def run(x_dev, nbin, delays, tsamp, t0, nu, nudot=0.0, nuddot=0.0, first=0):
    plan = Fold()
    plan.init(nbin, delays, tsamp, t0, nu, nudot, nuddot)
    shape = tuple(x_dev.shape[:-1]) + (nbin,)
    d_out = bf.asarray(np.full(shape, -7.0, np.float32), space='cuda')
    d_cnt = bf.asarray(np.full((x_dev.shape[0], nbin), -7, np.int32), space='cuda')
    plan.execute(x_dev, d_out, d_cnt, first=first)
    bf.device.stream_synchronize()
    return host(d_out), host(d_cnt), plan


def desc_delays(nchan, dm=30.0, f0=1500.0, df=-1.0):
    """Delays of a band whose channel 0 is the highest (negative df)."""
    f = f0 + df * np.arange(nchan)
    return dispersion_delays(f, dm, f.max())


CASES = {
    # name: (shape, nbin, tsamp, t0, nu, nudot, nuddot, first, delays)
    'batched_1000':    ((3, 4, 20000), 1000, 64e-6, 0.0, 1.7, 0.0, 0.0, 0, 'desc'),
    'nbin1':           ((2, 3000), 1, 1e-3, 0.3, 11.0, 0.0, 0.0, 5, 'desc'),
    'nbin7':           ((4, 2, 3001), 7, 1e-3, 0.3, 11.0, 0.0, 0.0, 77, 'desc'),
    'fast_700Hz':      ((4, 2, 50000), 1024, 64e-6, 0.0, 700.0, 0.0, 0.0, 0, 'desc'),
    'slow_1Hz_4096':   ((2, 1, 300000), 4096, 1e-6, 0.0, 1.0, 0.0, 0.0, 1000, 'zero'),
    'spin_terms':      ((3, 2, 40000), 256, 64e-6, 12.0, 30.0, -1e-3, 1e-5, 0, 'desc'),
    't0_plus_1e5':     ((2, 2, 30000), 1024, 64e-6, 1e5, 29.946923, -3.77e-10, 1e-20, 1 << 33, 'desc'),
    't0_minus_1e5':    ((2, 2, 30000), 1024, 64e-6, -1e5, 29.946923, -3.77e-10, 1e-20, 0, 'desc'),
    'ragged':          ((5, 1, 4097), 100, 3e-4, 0.0, 3.1, 0.0, 0.0, 3, 'desc'),
    'short':           ((3, 2, 17), 8, 1e-2, 0.0, 9.0, 0.0, 0.0, 0, 'desc'),
}


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['u8', 'u16', 'f32'])
@pytest.mark.parametrize('case', sorted(CASES))
def test_matches_oracle(case, dtype):
    shape, nbin, tsamp, t0, nu, nudot, nuddot, first, dk = CASES[case]
    rng = np.random.default_rng(abs(hash((case, dtype))) % (1 << 31))
    x = make_input(rng, dtype, shape)
    delays = desc_delays(shape[0]) if dk == 'desc' else np.zeros(shape[0])
    got, cnt, _ = run(bf.asarray(x, space='cuda'), nbin, delays, tsamp, t0, nu, nudot, nuddot, first)
    want, wcnt = ofold.fold(x, nbin, delays, tsamp, t0, nu, nudot, nuddot, first)
    assert np.array_equal(cnt, wcnt)
    check_sums(got, want, x, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['u8', 'u16', 'f32'])
def test_strided_and_offset_by_one(dtype):
    """Strided leading axes, a base one sample past a 16-byte boundary and
    strided output rows."""
    rng = np.random.default_rng(3)
    x = make_input(rng, dtype, (6, 3, 12001))
    d_big = bf.asarray(x, space='cuda')
    d_x = d_big[::2, 1:, 1:]
    xs = x[::2, 1:, 1:]
    delays = desc_delays(3)
    plan = Fold()
    plan.init(1000, delays, 64e-6, 0.5, 7.7)
    d_out = bf.zeros((3, 2, 2, 1000), 'f32', 'cuda')
    d_cnt = bf.zeros((3, 2, 1000), 'i32', 'cuda')
    plan.execute(d_x, d_out[:, :, 1, :], d_cnt[:, 1, :], first=9)
    bf.device.stream_synchronize()
    got, cnt = host(d_out), host(d_cnt)
    want, wcnt = ofold.fold(xs, 1000, delays, 64e-6, 0.5, 7.7, first=9)
    assert np.array_equal(cnt[:, 1], wcnt) and np.all(cnt[:, 0] == 0)
    check_sums(got[:, :, 1], want, xs, dtype)
    assert np.all(got[:, :, 0] == 0)


@pytest.mark.gpu
def test_nonfinite_rows_poison_only_their_bins():
    rng = np.random.default_rng(4)
    x = make_input(rng, 'f32', (2, 3, 5000))
    x[0, 1, 100] = np.nan
    x[1, 0, 2000] = np.inf
    x[1, 2, 10] = -np.inf
    x[1, 2, 4000] = np.inf
    delays = desc_delays(2)
    got, cnt, _ = run(bf.asarray(x, space='cuda'), 64, delays, 1e-3, 0.0, 1.3)
    want, wcnt = ofold.fold_nonfinite(x, 64, delays, 1e-3, 0.0, 1.3)
    assert np.array_equal(cnt, wcnt)
    assert np.sum(~np.isfinite(got)) == np.sum(~np.isfinite(want)) <= 4
    check_sums(got, want, np.where(np.isfinite(x), x, 0), 'f32')


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['u8', 'u16', 'f32'])
def test_accumulate_over_uneven_split(dtype):
    rng = np.random.default_rng(5)
    x = make_input(rng, dtype, (3, 2, 70001))
    delays = desc_delays(3)
    args = (512, delays, 64e-6, 3.0, 173.3, -2e-6, 0.0)
    whole, wcnt, _ = run(bf.asarray(x, space='cuda'), *args, first=1000)
    plan = Fold()
    plan.init(*args)
    d_out = bf.zeros((3, 2, 512), 'f32', 'cuda')
    d_cnt = bf.zeros((3, 512), 'i32', 'cuda')
    cuts = [0, 1, 18, 5003, 5004, 40000, 70001]
    for a, b in zip(cuts[:-1], cuts[1:]):
        plan.execute(bf.asarray(np.ascontiguousarray(x[..., a:b]), space='cuda'), d_out, d_cnt,
                     first=1000 + a, accumulate=a > 0)
    bf.device.stream_synchronize()
    got, cnt = host(d_out), host(d_cnt)
    assert np.array_equal(cnt, wcnt)
    want, ocnt = ofold.fold(x, *args, first=1000)
    assert np.array_equal(cnt, ocnt)
    if dtype == 'f32':
        # each call adds its fp64 partial to the f32 running sum: one f32
        # rounding per call, so a few ulp of the whole-stream sum
        err = np.abs(got.astype(np.float64) - want)
        assert np.all(err <= 6 * np.spacing(np.abs(want).astype(np.float32)) + 1e-9), err.max()
    else:
        assert np.array_equal(got.view(np.uint32), whole.view(np.uint32))


@pytest.mark.gpu
def test_repeatable_workspace_protocol_and_empty_calls():
    rng = np.random.default_rng(6)
    x = make_input(rng, 'f32', (4, 2, 100000))
    d_x = bf.asarray(x, space='cuda')
    plan = Fold()
    plan.init(1024, desc_delays(4), 64e-6, 0.0, 641.9)
    outs = [bf.zeros((4, 2, 1024), 'f32', 'cuda') for _ in range(3)]
    cnts = [bf.zeros((4, 1024), 'i32', 'cuda') for _ in range(3)]
    size = plan.get_workspace_size(d_x, outs[0], cnts[0])       # (NULL, &size): query only
    bf.device.stream_synchronize()
    assert size > 0 and np.all(host(outs[0]) == 0) and np.all(host(cnts[0]) == 0)
    plan.execute(d_x, outs[0], cnts[0])                          # (NULL, NULL): library-managed
    plan.execute(d_x, outs[1], cnts[1])
    ws = bf.empty((size,), dtype='u8', space='cuda')
    plan.execute_workspace(d_x, outs[2], cnts[2], ws.ctypes.data, size)   # (ptr, &size)
    bf.device.stream_synchronize()
    a = [host(o) for o in outs]
    assert np.array_equal(a[0].view(np.uint32), a[1].view(np.uint32))
    assert np.array_equal(a[0].view(np.uint32), a[2].view(np.uint32))
    for c in cnts[1:]:
        assert np.array_equal(host(c), host(cnts[0]))
    small = _bf.BFsize(size - 1)
    st = _bf.bfFoldExecute(plan.obj, d_x.as_BFarray(), 0, outs[1].as_BFarray(), cnts[1].as_BFarray(), 0,
                           ctypes.c_void_p(ws.ctypes.data), ctypes.byref(small))
    assert st == _bf.BF_STATUS_INSUFFICIENT_STORAGE
    st = _bf.bfFoldExecute(plan.obj, d_x.as_BFarray(), 0, outs[1].as_BFarray(), cnts[1].as_BFarray(), 0,
                           ctypes.c_void_p(ws.ctypes.data), None)
    assert st == _bf.BF_STATUS_INVALID_ARGUMENT
    # ntime 0 and an empty batch axis: accumulate keeps, overwrite zeroes
    for shape in ((4, 2, 0), (4, 0, 100)):
        d_e = bf.zeros(shape, 'f32', 'cuda')
        o = bf.asarray(np.full(shape[:-1] + (1024,), 5.0, np.float32), space='cuda')
        n = bf.asarray(np.full((4, 1024), 5, np.int32), space='cuda')
        plan.execute(d_e, o, n, accumulate=True)
        bf.device.stream_synchronize()
        assert np.all(host(o) == 5.0) and np.all(host(n) == 5)
        plan.execute(d_e, o, n)
        bf.device.stream_synchronize()
        assert np.all(host(o) == 0.0) and np.all(host(n) == 0)


def status(plan, x, out, cnt, acc=0):
    return _bf.bfFoldExecute(plan.obj if plan is not None else None,
                             x.as_BFarray() if x is not None else None, 0,
                             out.as_BFarray() if out is not None else None,
                             cnt.as_BFarray() if cnt is not None else None, acc, None, None)


@pytest.mark.gpu
def test_error_statuses():
    S = _bf
    plan = Fold()
    d_x = bf.zeros((4, 2, 1000), 'u8', 'cuda')
    d_o = bf.zeros((4, 2, 64), 'f32', 'cuda')
    d_n = bf.zeros((4, 64), 'i32', 'cuda')
    assert status(plan, d_x, d_o, d_n) == S.BF_STATUS_INVALID_STATE
    plan.init(64, np.zeros(4), 1e-3, 0.0, 1.0)
    assert status(plan, d_x, d_o, d_n) == S.BF_STATUS_SUCCESS
    assert status(None, d_x, d_o, d_n) == S.BF_STATUS_INVALID_HANDLE
    assert status(plan, None, d_o, d_n) == S.BF_STATUS_INVALID_POINTER
    assert status(plan, d_x, None, d_n) == S.BF_STATUS_INVALID_POINTER
    assert status(plan, d_x, d_o, None) == S.BF_STATUS_INVALID_POINTER
    assert status(plan, bf.zeros((4, 2, 1000), 'u8'), d_o, d_n) == S.BF_STATUS_UNSUPPORTED_SPACE
    assert status(plan, d_x, bf.zeros((4, 2, 64), 'f32'), d_n) == S.BF_STATUS_UNSUPPORTED_SPACE
    assert status(plan, d_x, d_o, bf.zeros((4, 64), 'i32')) == S.BF_STATUS_UNSUPPORTED_SPACE
    for dt in ('i8', 'i16', 'f64', 'cf32', 'ci8', 'i32'):
        assert status(plan, bf.zeros((4, 2, 1000), dt, 'cuda'), d_o, d_n) == S.BF_STATUS_UNSUPPORTED_DTYPE, dt
    for dt in ('f64', 'i32', 'cf32'):
        assert status(plan, d_x, bf.zeros((4, 2, 64), dt, 'cuda'), d_n) == S.BF_STATUS_UNSUPPORTED_DTYPE, dt
    for dt in ('u32', 'f32', 'i16'):
        assert status(plan, d_x, d_o, bf.zeros((4, 64), dt, 'cuda')) == S.BF_STATUS_UNSUPPORTED_DTYPE, dt
    for shape in ((4, 2, 63), (4, 3, 64), (3, 2, 64), (4, 2, 64, 1), (4, 64)):
        assert status(plan, d_x, bf.zeros(shape, 'f32', 'cuda'), d_n) == S.BF_STATUS_INVALID_SHAPE, shape
    for shape in ((4, 63), (3, 64), (4, 64, 1), (256,)):
        assert status(plan, d_x, d_o, bf.zeros(shape, 'i32', 'cuda')) == S.BF_STATUS_INVALID_SHAPE, shape
    assert status(plan, bf.zeros((3, 2, 1000), 'u8', 'cuda'), bf.zeros((3, 2, 64), 'f32', 'cuda'),
                  d_n) == S.BF_STATUS_INVALID_SHAPE                  # nchan differs from the plan
    assert status(plan, bf.zeros((1000,), 'u8', 'cuda'), bf.zeros((64,), 'f32', 'cuda'),
                  d_n) == S.BF_STATUS_INVALID_SHAPE                  # no channel axis
    wide = bf.zeros((4, 2, 2000), 'u8', 'cuda')
    assert status(plan, wide[:, :, ::2], d_o, d_n) == S.BF_STATUS_UNSUPPORTED_STRIDE
    wo = bf.zeros((4, 2, 128), 'f32', 'cuda')
    assert status(plan, d_x, wo[:, :, ::2], d_n) == S.BF_STATUS_UNSUPPORTED_STRIDE
    wn = bf.zeros((4, 128), 'i32', 'cuda')
    assert status(plan, d_x, d_o, wn[:, ::2]) == S.BF_STATUS_UNSUPPORTED_STRIDE
    bf.device.stream_synchronize()


@pytest.mark.gpu
def test_kernel_path():
    from kernel_trace import device_kernels
    rng = np.random.default_rng(7)
    plan = Fold()
    plan.init(256, desc_delays(4), 64e-6, 0.0, 1.4)
    d_o = bf.zeros((4, 2, 256), 'f32', 'cuda')
    d_n = bf.zeros((4, 256), 'i32', 'cuda')
    for dt in ('u8', 'u16', 'f32'):
        d_x = bf.asarray(make_input(rng, dt, (4, 2, 30000)), space='cuda')
        plan.execute(d_x, d_o, d_n)                # workspace outside the trace
        names = device_kernels(lambda: plan.execute(d_x, d_o, d_n, accumulate=True))
        assert len(names) == 2, names
        assert 'fold_kernel' in names[0] and 'fold_finish_kernel' in names[1], names


# ------------------------------------------------------------------ pipelines
P_NCHAN, P_F0, P_DF, P_DM = 4, 400.78125, 1.5625, 1.0      # channels 400.78 .. 405.47 MHz
P_NBLOCK, P_AMP, P_NBIN = 8, 400., 64
P_PERIOD = 611.37                                          # samples per turn


def pulse_train_voltages(seed=17):
    """ci8 [block, chan, ntime, pol] of a GUPPI RAW file: Gaussian noise of
    sigma 8 per component plus an impulse every P_PERIOD samples (first at
    T0), shifted per channel by its top-edge delay relative to the highest
    channel and then dispersed inside each channel."""
    from oracle import coherent_dedisp as ocd
    m = dispersion_overlap(P_NCHAN, P_F0, P_DF, P_DM)
    nfft = default_nfft(m)
    ntime = 2 * (nfft - m)
    total = P_NBLOCK * ntime
    rng = np.random.default_rng(seed)
    tops = P_F0 + P_DF * np.arange(P_NCHAN) + P_DF / 2
    shift = KDM * P_DM * (tops ** -2 - tops[-1] ** -2) * P_DF * 1e6
    t0 = 37.0
    imp = np.zeros((P_NCHAN, 2, total), complex)
    k = 0
    while t0 + k * P_PERIOD + shift.max() < total - 1:
        for c in range(P_NCHAN):
            imp[c, :, int(np.rint(t0 + k * P_PERIOD + shift[c]))] = P_AMP * np.array([1.0, 0.6 - 0.5j])
        k += 1
    v = ocd.disperse(imp, P_F0, P_DF, P_DM) + 8 * (rng.normal(size=imp.shape) + 1j * rng.normal(size=imp.shape))
    re = np.clip(np.rint(v.real), -127, 127).astype(np.int8)
    im = np.clip(np.rint(v.imag), -127, 127).astype(np.int8)
    data = np.stack([re, im], -1).reshape(P_NCHAN, 2, P_NBLOCK, ntime, 2).transpose(2, 0, 3, 1, 4)
    return np.ascontiguousarray(data), t0, k, ntime


def write_guppi(path, data):
    from bifrost_b200 import guppi_raw
    nblock, nchan, ntime = data.shape[:3]
    with open(path, 'wb') as f:
        for b in range(nblock):
            hdr = dict(BACKEND='GUPPI', TELESCOP='GBT', SRC_NAME='FAKE',
                       OBSFREQ=P_F0 + 0.5 * (nchan - 1) * P_DF, OBSBW=P_DF * nchan,
                       OBSNCHAN=nchan, NPOL=4, NBITS=8, BLOCSIZE=nchan * ntime * 4, PKTIDX=b * 16,
                       PKTSIZE=8192, STT_IMJD=58849, STT_SMJD=43200, RA=53.2475, DEC=54.5787, CHAN_DM=0.0)
            guppi_raw.write_header(hdr, f)
            data[b].tofile(f)


def check_subints(subs, power, head, nbin, nu, nsub, tsamp, delays):
    """Every emitted subintegration is the oracle's mean profile of the power
    stream over its samples (the f32 running sum is rounded once per gulp:
    a relative 1e-6)."""
    nchan = power.shape[0]
    assert len(subs) == power.shape[-1] // nsub and len(subs) >= 1
    for s, got in enumerate(subs):
        seg = power[..., s * nsub:(s + 1) * nsub]
        sums, counts = ofold.fold(seg, nbin, delays, tsamp, 0.0, nu, first=s * nsub)
        cshape = (nchan,) + (1,) * (seg.ndim - 2) + (nbin,)
        want = np.where(counts.reshape(cshape) > 0, sums / np.maximum(counts, 1).reshape(cshape), 0.0)
        got = got.reshape(want.shape)
        assert np.all(np.abs(got - want) <= 1e-6 * np.abs(want) + 1e-9), (s, np.abs(got - want).max())


@pytest.mark.gpu
def test_coherent_chain_folds_pulse_train(tmp_path):
    from bifrost_b200 import blocks, views
    from bifrost_b200.pipeline import Pipeline
    data, t0, nturn, ntime = pulse_train_voltages()
    assert nturn >= 20
    path = str(tmp_path / 'psr.raw')
    write_guppi(path, data)
    tsamp = 1.0 / (P_DF * 1e6)
    nu = 1.0 / (P_PERIOD * tsamp)
    power, subs, heads = [], [], []
    with Pipeline() as p:
        b = blocks.read_guppi_raw([path])
        b = blocks.copy(b, space='cuda')
        b = blocks.transpose(b, ['freq', 'pol', 'time', 'fine_time'])
        b = views.merge_axes(b, 'time', 'fine_time')
        b = blocks.coherent_dedisp(b, P_DM)
        d = blocks.detect(b, 'stokes_i')
        blocks.callback_sink(blocks.copy(d, space='system'), None, lambda q: power.append(np.array(q.data)))
        f = blocks.fold(d, P_NBIN, nu, dm=None, tsubint=2 * ntime * tsamp)
        blocks.callback_sink(blocks.copy(f, space='system'), lambda q: heads.append(deepcopy(q.header)),
                             lambda q: subs.extend(np.array(q.data)))
        p.run()
    head = heads[0]
    pw = np.concatenate(power, axis=-1)
    nsub = head['fold_nsamp_sub']
    assert nsub == 2 * ntime and head['fold_dm'] == P_DM
    assert head['_tensor']['labels'][0] == 'time' and head['_tensor']['labels'][-1] == 'phase'
    tops = P_F0 + P_DF * np.arange(P_NCHAN) + P_DF / 2
    delays = dispersion_delays(tops, P_DM, tops[-1])
    assert head['fold_fref'] == tops[-1]
    check_subints(subs, pw, head, P_NBIN, nu, nsub, tsamp, delays)
    prof = np.mean([s.reshape(P_NCHAN, -1, P_NBIN)[:, 0] for s in subs], axis=0)
    peak = int(math.floor((t0 / P_PERIOD) % 1.0 * P_NBIN))
    for c in range(P_NCHAN):
        assert int(np.argmax(prof[c])) == peak, (c, np.argmax(prof[c]), peak)
        assert prof[c].max() > 5 * np.median(prof[c]), (c, prof[c].max(), np.median(prof[c]))


F_NCHAN, F_F0, F_DF, F_TSAMP, F_GULP = 32, 1500.0, -1.0, 256e-6, 4096
F_DM, F_NU, F_NBIN = 50.0, 1.0 / (173.31 * 256e-6), 32


@pytest.mark.gpu
def test_filterbank_folds_pulse_train():
    from bifrost_b200 import blocks
    from bifrost_b200.pipeline import Pipeline
    rng = np.random.default_rng(18)
    ntime = 6 * F_GULP + 1000                                   # a partial last subint is not emitted
    freqs = F_F0 + F_DF * np.arange(F_NCHAN)
    delays = dispersion_delays(freqs, F_DM, freqs.max())
    x = rng.normal(64, 8, size=(F_NCHAN, ntime))
    t = np.arange(ntime) * F_TSAMP
    phase = ((t[None, :] - delays[:, None]) * F_NU) % 1.0
    x += 60 * (np.abs(phase - 0.3) < 0.01)
    x = np.clip(np.rint(x), 0, 255).astype(np.uint8)
    hdr = {'_tensor': {'dtype': 'u8', 'shape': [-1, F_NCHAN], 'labels': ['time', 'freq'],
                       'scales': [[1.6e9, F_TSAMP], [F_F0, F_DF]], 'units': ['s', 'MHz']},
           'name': 'fil', 'gulp_nframe': F_GULP}
    subs = []
    with Pipeline() as p:
        src = blocks.array_source(np.ascontiguousarray(x.T), hdr, gulp_nframe=F_GULP)
        b = blocks.copy(src, space='cuda')
        b = blocks.transpose(b, ['freq', 'time'])
        f = blocks.fold(b, F_NBIN, F_NU, dm=F_DM, tsubint=2 * F_GULP * F_TSAMP)
        blocks.callback_sink(blocks.copy(f, space='system'), None, lambda q: subs.extend(np.array(q.data)))
        p.run()
    assert len(subs) == 3
    check_subints(subs, x, None, F_NBIN, F_NU, 2 * F_GULP, F_TSAMP, delays)
    prof = np.mean(subs, axis=0)
    peak = int(0.3 * F_NBIN)
    for c in range(F_NCHAN):
        assert abs(int(np.argmax(prof[c])) - peak) <= 1, (c, np.argmax(prof[c]))
        assert prof[c].max() > np.median(prof[c]) + 5, (c, prof[c].max(), np.median(prof[c]))
