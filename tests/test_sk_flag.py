"""bfSkFlag*: RFI excision by windowed spectral kurtosis.

CPU: the oracle (oracle/sk_flag.py) against a per-window loop, a Monte Carlo
of the estimator's mean and variance, exact edge cases, the thresholds, the
block header and Init's argument checks.  GPU: bfSkFlagExecute against the
oracle (bit for bit for u8 / u16) on batched / strided / offset / in-place /
short-window inputs, NaN rows, the config-2 filterbank shape, its statuses and
workspace protocol, the kernel path, and a u8 filterbank with RFI through
copy -> transpose -> sk_flag -> fdmt -> pulse_search."""
import ctypes
import os
import sys
from copy import deepcopy

import numpy as np
import pytest

import bifrost_b200 as bf
from bifrost_b200.libbifrost import _bf
from bifrost_b200.blocks.sk_flag import sk_flag_header
from bifrost_b200.sk_flag import SkFlag, sk_thresholds, sk_variance, sk_nwindow
from oracle import sk_flag as osk

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------ oracle (CPU)
def loop_sk_flag(x, M, N, d, lo, hi):
    """The definition, one window at a time with Python ints and floats."""
    x = np.asarray(x)
    ntime = x.shape[-1]
    nwin = -(-ntime // M)
    y = x.copy()
    sk = np.zeros(x.shape[:-1] + (nwin,))
    flags = np.zeros(x.shape[:-1] + (nwin,), bool)
    integer = x.dtype != np.float32
    for r in np.ndindex(*x.shape[:-1]):
        tot, cnt = 0.0, 0
        for j in range(nwin):
            w = x[r][j * M:min((j + 1) * M, ntime)]
            m = len(w)
            if integer:
                s1 = float(sum(int(v) for v in w))
                s2 = float(sum(int(v) * int(v) for v in w))
            else:
                s1 = sum(float(v) for v in w)
                s2 = sum(float(v) * float(v) for v in w)
            a = ((m * N) * d + 1) / (m - 1) if m > 1 else float('inf')
            with np.errstate(all='ignore'):
                k = float(np.float64(a) * (np.float64(m * s2) / np.float64(s1 * s1) - 1.0))
            sk[r + (j,)] = k
            flags[r + (j,)] = not (lo <= k <= hi)
            if not flags[r + (j,)]:
                tot += s1
                cnt += m
        fill = tot / cnt if cnt else 0.0
        fv = np.float32(fill) if not integer else np.rint(fill).astype(x.dtype)
        for j in range(nwin):
            if flags[r + (j,)]:
                y[r][j * M:(j + 1) * M] = fv
    return y, sk, flags


def power(rng, shape, dtype, k=4.0, scale=8.0, rfi=0.05):
    """Gamma(k, scale) power in `dtype` with about `rfi` of the rows' 64-sample
    stretches given a constant or a spike."""
    x = rng.gamma(k, scale, size=shape)
    flat = x.reshape(-1, shape[-1])
    for _ in range(max(1, int(rfi * flat.size / 64))):
        r, t = rng.integers(flat.shape[0]), rng.integers(shape[-1])
        if rng.random() < 0.5:
            flat[r, t:t + 64] = k * scale * 2
        else:
            flat[r, t] += 12 * k * scale
    if dtype == np.float32:
        return x.astype(np.float32)
    top = np.iinfo(dtype).max
    return np.clip(np.rint(x), 0, top).astype(dtype)


@pytest.mark.parametrize('seed', range(6))
def test_oracle_equals_loop(seed):
    rng = np.random.default_rng(seed)
    dtype = (np.uint8, np.uint16, np.float32)[seed % 3]
    M = int(rng.integers(2, 40))
    ntime = int(rng.integers(1, 5)) * M + int(rng.integers(0, M))      # often a short last window
    N, d = int(rng.integers(1, 5)), float(rng.choice([0.5, 1.0, 2.0]))
    scale = 1000. if dtype == np.uint16 else 8.
    x = power(rng, (2, 3, ntime), dtype, scale=scale, rfi=0.2)
    lo, hi = sk_thresholds(M, N, d)
    y, sk32, flags, sk64, _ = osk.sk_flag(x, M, N, d, lo, hi)
    wy, wsk, wflags = loop_sk_flag(x, M, N, d, lo, hi)
    np.testing.assert_array_equal(flags, wflags)
    if dtype == np.float32:
        np.testing.assert_allclose(sk64, wsk, rtol=1e-12, atol=0)
        np.testing.assert_allclose(y, wy, rtol=1e-6, atol=0)
    else:
        np.testing.assert_array_equal(sk64, wsk)
        np.testing.assert_array_equal(y, wy)
    assert y.dtype == x.dtype and sk32.dtype == np.float32


@pytest.mark.parametrize('M,N,d', [(64, 1, 1.0), (16, 4, 1.0), (256, 1, 0.5)])
def test_monte_carlo_mean_and_variance(M, N, d):
    rng = np.random.default_rng(M * 10 + N)
    nwin, chunk = 200000, 20000
    ks = []
    for _ in range(nwin // chunk):
        x = rng.standard_gamma(N * d, size=(chunk, M), dtype=np.float32)
        s1, s2, m = osk.window_sums(x, M)
        ks.append(osk.sk(s1, s2, m, N, d)[:, 0])
    k = np.concatenate(ks)
    var = sk_variance(M, N, d)
    assert abs(k.mean() - 1) < 5 * np.sqrt(var / nwin), (k.mean(), var)
    assert abs(k.var() / var - 1) < 0.03, (k.var(), var)


def test_exact_cases():
    M, lo, hi = 16, 1e-6, 1.0
    rng = np.random.default_rng(3)
    x = rng.integers(8, 13, size=(1, 5 * M + 1)).astype(np.uint8)   # sk about 0.02: clean
    x[0, M:2 * M] = 7                                    # constant: sk == 0, flagged low
    x[0, 2 * M:3 * M] = 0                                # zero: 0 / 0 = NaN, flagged
    x[0, 3 * M + 5] = 250                                # spike: flagged high
    y, _, flags, k, fill = osk.sk_flag(x, M, 1, 1.0, lo, hi)
    assert k[0, 1] == 0 and np.isnan(k[0, 2]) and k[0, 3] > hi
    assert np.isnan(k[0, 5])                             # the last window has m = 1
    assert lo < k[0, 0] < hi and lo < k[0, 4] < hi
    assert list(flags[0]) == [False, True, True, True, False, True]
    clean = np.r_[x[0, :M], x[0, 4 * M:5 * M]].astype(np.int64)
    assert fill[0] == clean.sum() / (2 * M)
    per = np.repeat(flags[0], M)[:x.shape[1]]
    assert np.all(y[0, per] == np.rint(fill[0])) and np.array_equal(y[0, ~per], x[0, ~per])


def test_fill_rounds_half_to_even():
    M = 16
    for lowv, want in ((2, 2), (3, 4)):                  # clean means 2.5 and 3.5
        x = np.empty((1, 3 * M), np.uint8)
        x[0, :2 * M] = np.tile([lowv, lowv + 1], M)
        x[0, 2 * M:] = 200                               # constant: flagged
        y, _, flags, _, fill = osk.sk_flag(x, M, 1, 1.0, 0.01, 10.)
        assert list(flags[0]) == [False, False, True] and fill[0] == lowv + 0.5
        assert np.all(y[0, 2 * M:] == want)
    x = np.full((1, 3 * M), 1.0, np.float32)             # f32: round to nearest even of fp64
    x[0, :M] = np.tile(np.float32([1.0, 2.0]), M // 2)
    y, _, flags, _, fill = osk.sk_flag(x, M, 1, 1.0, 0.01, 10.)
    assert np.all(y[0, M:] == np.float32(fill[0])) and fill[0] == 1.5


def test_all_flagged_row_fills_zero():
    x = np.full((2, 100), 17, np.uint16)
    x[1] = np.arange(100) % 7 + 1
    y, _, flags, _, fill = osk.sk_flag(x, 10, 1, 1.0, 0.9, 1.1)
    assert flags[0].all() and np.all(y[0] == 0) and fill[0] == 0
    y, _, flags, _, _ = osk.sk_flag(np.zeros((1, 64), np.float32), 8, 1, 1.0, 0.5, 1.5)
    assert flags.all() and np.all(y == 0)


def test_one_sample_last_window_is_flagged():
    rng = np.random.default_rng(4)
    for dtype in (np.uint8, np.uint16, np.float32):
        x = power(rng, (3, 4 * 32 + 1), dtype, rfi=0)
        _, _, flags, k, _ = osk.sk_flag(x, 32, 1, 1.0, -1e300, 1e300)
        assert np.all(flags[:, -1]) and np.all(np.isnan(k[:, -1])) and not flags[:, :-1].any()


def test_thresholds():
    lo, hi = sk_thresholds(256, 4, 1.0, 3.0)
    v = 2 * 256 ** 2 * 4 * 5 / (255 * 1026 * 1027)
    assert np.isclose(hi - 1, 3 * np.sqrt(v), rtol=1e-14) and np.isclose(1 - lo, 3 * np.sqrt(v), rtol=1e-14)
    lo, hi = sk_thresholds(64, sigma=2.0)
    v = 2 * 64 ** 2 * 2 / (63 * 66 * 67)
    assert np.isclose(hi, 1 + 2 * np.sqrt(v)) and np.isclose(lo, 1 - 2 * np.sqrt(v))
    assert sk_nwindow(1000, 256) == 4 and sk_nwindow(1024, 256) == 4 and sk_nwindow(0, 256) == 0


def filterbank_header(nchan=256, dtype='u8', gulp=4096):
    return {'_tensor': {'dtype': dtype, 'shape': [nchan, -1], 'labels': ['freq', 'time'],
                        'scales': [[1200., 0.5], [0, 1e-3]], 'units': ['MHz', 's']},
            'name': 'fil', 'gulp_nframe': gulp}


def test_block_header():
    ihdr = filterbank_header()
    keep = deepcopy(ihdr)
    ohdr = sk_flag_header(ihdr, 256, 4, 1.0, 3.0)
    assert ihdr == keep
    assert ohdr['_tensor'] == ihdr['_tensor']
    assert ohdr['sk_window'] == 256 and ohdr['sk_nacc'] == 4 and ohdr['sk_shape'] == 1.0
    assert ohdr['sk_thresholds'] == list(sk_thresholds(256, 4, 1.0, 3.0))
    for dt in ('u16', 'f32'):
        assert sk_flag_header(filterbank_header(dtype=dt), 64)['_tensor']['dtype'] == dt
    for dt in ('i8', 'i16', 'cf32', 'f64'):
        with pytest.raises(TypeError):
            sk_flag_header(filterbank_header(dtype=dt), 64)
    with pytest.raises(KeyError):
        sk_flag_header({'_tensor': dict(ihdr['_tensor'], shape=[-1, 256], labels=['time', 'freq'])}, 64)


@pytest.mark.parametrize('args', [(1, 1, 1.0, 0.5, 1.5), ((1 << 20) + 1, 1, 1.0, 0.5, 1.5),
                                  (0, 1, 1.0, 0.5, 1.5), (64, 0, 1.0, 0.5, 1.5), (64, 1, 0.0, 0.5, 1.5),
                                  (64, 1, -1.0, 0.5, 1.5), (64, 1, float('nan'), 0.5, 1.5),
                                  (64, 1, float('inf'), 0.5, 1.5), (64, 1, 1.0, 1.5, 1.5),
                                  (64, 1, 1.0, 1.6, 1.5), (64, 1, 1.0, float('-inf'), 1.5),
                                  (64, 1, 1.0, 0.5, float('inf')), (64, 1, 1.0, float('nan'), 1.5)])
def test_init_rejects_bad_arguments(args):
    plan = SkFlag()
    window, nacc, shape, lo, hi = args
    with pytest.raises(RuntimeError, match='INVALID_ARGUMENT'):
        plan.init(window, nacc, shape, lo, hi)


def test_init_accepts_limits():
    plan = SkFlag()
    plan.init(2, 1, 1.0, -1.0, 1.0)
    plan.init(1 << 20, 1 << 30, 1e-3)
    assert (plan.lo, plan.hi) == sk_thresholds(1 << 20, 1 << 30, 1e-3)


# ------------------------------------------------------------------ GPU
def host(d):
    return np.asarray(d.copy('system'))


def nan_equal(a, b):
    """Bitwise equal f32 arrays, NaN equal to NaN whatever its payload."""
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def changed_windows(x, y, M):
    """Windows where y differs from x anywhere: the windows the library flagged,
    as long as no flagged window already equalled the fill everywhere."""
    ntime = x.shape[-1]
    nwin = -(-ntime // M)
    diff = (x != y).reshape(-1, ntime)
    pad = np.zeros((diff.shape[0], nwin * M - ntime), bool)
    return np.concatenate([diff, pad], axis=1).reshape(x.shape[:-1] + (nwin, M)).any(axis=-1)


def run(d_x, M, N=1, d=1.0, lo=None, hi=None, d_y=None, with_sk=True):
    lead, ntime = d_x.shape[:-1], d_x.shape[-1]
    if d_y is None:
        d_y = bf.zeros(d_x.shape, d_x.dtype, 'cuda')
    d_k = bf.zeros(lead + (sk_nwindow(ntime, M),), 'f32', 'cuda') if with_sk else None
    plan = SkFlag()
    plan.init(M, N, d, lo, hi)
    plan.execute(d_x, d_y, d_k)
    bf.device.stream_synchronize()
    return d_y, d_k, plan


def check_exact(x, y, k, M, N, d, lo, hi):
    wy, wk, wflags, _, _ = osk.sk_flag(x, M, N, d, lo, hi)
    assert np.array_equal(y, wy)
    assert nan_equal(k, wk)
    assert np.array_equal(changed_windows(x, y, M), changed_windows(x, wy, M))
    assert np.array_equal(changed_windows(x, wy, M), wflags)         # every flag is visible in y
    return wflags


INT_CASES = {
    # name: (lead, ntime, M, N)
    'batch':      ((2, 3, 5), 3000, 256, 4),
    'nwin1':      ((7,), 1000, 4096, 1),
    'last_m1':    ((6,), 5 * 64 + 1, 64, 1),
    'last_mM-1':  ((6,), 6 * 64 - 1, 64, 2),
    'small_M':    ((5,), 999, 3, 1),
    'wide_M':     ((3,), 300000, 1 << 17, 4),
}


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['u8', 'u16'])
@pytest.mark.parametrize('name', sorted(INT_CASES))
def test_integer_matches_oracle(name, dtype):
    lead, ntime, M, N = INT_CASES[name]
    rng = np.random.default_rng(sorted(INT_CASES).index(name))
    npdt = np.uint8 if dtype == 'u8' else np.uint16
    x = power(rng, lead + (ntime,), npdt, k=float(N), scale=8. if dtype == 'u8' else 1000.)
    lo, hi = sk_thresholds(M, N)
    d_y, d_k, _ = run(bf.asarray(x, space='cuda'), M, N, 1.0, lo, hi)
    flags = check_exact(x, host(d_y), host(d_k), M, N, 1.0, lo, hi)
    assert flags.any()
    if flags.size > 50:
        assert not flags.all()


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['u8', 'u16', 'f32'])
def test_row_pitch_offset_base_and_output_strides(dtype):
    rng = np.random.default_rng(5)
    npdt = {'u8': np.uint8, 'u16': np.uint16, 'f32': np.float32}[dtype]
    ntime, M, N = 5000, 256, 4
    big = power(rng, (2, 7, ntime + 37), npdt, scale=8. if dtype != 'u16' else 1000.)
    d_big = bf.asarray(big, space='cuda')
    view = d_big[:, 1:, 1:1 + ntime]                           # row pitch ntime + 37, base + 1 element
    x = big[:, 1:, 1:1 + ntime]
    d_ybig = bf.zeros((2, 6, ntime + 100), dtype, 'cuda')
    yview = d_ybig[:, :, 3:3 + ntime]                          # its own pitch and offset
    nwin = sk_nwindow(ntime, M)
    d_kbig = bf.zeros((2, 6, nwin + 5), 'f32', 'cuda')
    kview = d_kbig[:, :, 2:2 + nwin]
    lo, hi = sk_thresholds(M, N)
    plan = SkFlag()
    plan.init(M, N, 1.0, lo, hi)
    plan.execute(view, yview, kview)
    bf.device.stream_synchronize()
    ybig, kbig = host(d_ybig), host(d_kbig)
    y, k = ybig[:, :, 3:3 + ntime], kbig[:, :, 2:2 + nwin]
    assert np.all(ybig[:, :, :3] == 0) and np.all(ybig[:, :, 3 + ntime:] == 0)
    assert np.all(kbig[:, :, :2] == 0) and np.all(kbig[:, :, 2 + nwin:] == 0)
    if dtype == 'f32':
        check_f32(x, y, k, M, N, 1.0, lo, hi)
    else:
        check_exact(x, y, k, M, N, 1.0, lo, hi)
    # in place on the strided, offset view: the same result, the padding untouched
    plan.execute(view, view)
    bf.device.stream_synchronize()
    after = host(d_big)
    assert np.array_equal(after[:, 1:, 1:1 + ntime], y)
    assert np.array_equal(after[:, 0], big[:, 0]) and np.array_equal(after[:, :, 0], big[:, :, 0])
    assert np.array_equal(after[:, :, 1 + ntime:], big[:, :, 1 + ntime:])


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['u8', 'u16', 'f32'])
def test_in_place(dtype):
    rng = np.random.default_rng(6)
    npdt = {'u8': np.uint8, 'u16': np.uint16, 'f32': np.float32}[dtype]
    M, N = 64, 1
    x = power(rng, (9, 64 * 50 + 7), npdt, scale=8. if dtype != 'u16' else 1000.)
    lo, hi = sk_thresholds(M, N)
    d_x = bf.asarray(x, space='cuda')
    d_y, d_k, _ = run(d_x, M, N, 1.0, lo, hi, d_y=d_x)
    y, k = host(d_x), host(d_k)
    if dtype == 'f32':
        check_f32(x, y, k, M, N, 1.0, lo, hi)
    else:
        check_exact(x, y, k, M, N, 1.0, lo, hi)


def check_f32(x, y, k, M, N, d, lo, hi):
    wy, wk, wflags, wk64, fill = osk.sk_flag(x, M, N, d, lo, hi)
    fin = np.isfinite(wk64)
    rel = np.abs(wk64[fin] - np.array([lo, hi])[:, None]).min(axis=0) / np.maximum(np.abs(wk64[fin]), 1e-300)
    assert np.all(rel > 1e-9), "an oracle sk lies within 1e-9 of a threshold: flags not comparable"
    flags = changed_windows(x, y, M)
    assert np.array_equal(flags, wflags)
    per = np.repeat(wflags, M, axis=-1)[..., :x.shape[-1]]
    assert np.array_equal(y[~per].view(np.uint32), x[~per].view(np.uint32))        # clean: bit for bit
    ulp = np.abs(y.view(np.int32).astype(np.int64) - wy.view(np.int32).astype(np.int64))
    assert ulp[per].max(initial=0) <= 1                                            # fill within 1 ulp
    assert np.array_equal(np.isnan(k), np.isnan(wk))
    ok = ~np.isnan(wk)
    np.testing.assert_allclose(k[ok], wk64[ok], rtol=1e-6, atol=0)


F32_CASES = {
    'batch':   ((2, 3, 5), 3000, 256, 4, 1.0),
    'last_m1': ((4,), 3 * 100 + 1, 100, 1, 0.5),
    'nwin1':   ((6,), 700, 1024, 2, 1.0),
    'small_M': ((3,), 1001, 2, 1, 1.0),
}


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(F32_CASES))
def test_f32_matches_oracle(name):
    lead, ntime, M, N, d = F32_CASES[name]
    rng = np.random.default_rng(20 + sorted(F32_CASES).index(name))
    x = power(rng, lead + (ntime,), np.float32, k=N * d, scale=3.)
    lo, hi = sk_thresholds(M, N, d)
    d_y, d_k, _ = run(bf.asarray(x, space='cuda'), M, N, d, lo, hi)
    check_f32(x, host(d_y), host(d_k), M, N, d, lo, hi)


@pytest.mark.gpu
def test_nonfinite_row_leaves_other_rows_alone():
    rng = np.random.default_rng(7)
    M, N = 128, 1
    x = power(rng, (6, 3000), np.float32, k=1.0, scale=2.)
    x[2, 1700] = np.nan
    x[4, 10] = np.inf
    x[4, 2000] = -np.inf
    lo, hi = sk_thresholds(M, N)
    d_y, d_k, _ = run(bf.asarray(x, space='cuda'), M, N, 1.0, lo, hi)
    y, k = host(d_y), host(d_k)
    assert np.isnan(k[2, 1700 // M]) and np.isnan(k[4, 0]) and np.isnan(k[4, 2000 // M])
    assert np.all(np.isfinite(y))
    check_f32(x, y, k, M, N, 1.0, lo, hi)


def config2_filterbank(nchan=4096, ntime=131072, seed=8):
    """u8 Gamma(4, 8) power with about 3 % of its 256-sample windows corrupted,
    drawn on the device (torch) for speed."""
    import torch
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.empty(nchan, ntime, device='cuda').exponential_(generator=g)
    for _ in range(3):
        x += torch.empty(nchan, ntime, device='cuda').exponential_(generator=g)
    x = x * 8
    nwin = ntime // 256
    bad = torch.rand(nchan, nwin, device='cuda', generator=g) < 0.03
    xw = x.view(nchan, nwin, 256)
    xw[..., 100:104] += 150 * bad[..., None]
    return torch.clamp(torch.round(x), 0, 255).to(torch.uint8).cpu().numpy()


@pytest.mark.gpu
def test_config2_shape_and_repeatability():
    M, N = 256, 4
    x = config2_filterbank()
    lo, hi = sk_thresholds(M, N)
    d_x = bf.asarray(x, space='cuda')
    d_y, d_k, plan = run(d_x, M, N, 1.0, lo, hi)
    y1, k1 = host(d_y), host(d_k)
    plan.execute(d_x, d_y, d_k)
    bf.device.stream_synchronize()
    assert np.array_equal(host(d_y), y1) and np.array_equal(host(d_k).view(np.uint32), k1.view(np.uint32))
    nflag = 0
    for r0 in range(0, x.shape[0], 256):
        sl = slice(r0, r0 + 256)
        wy, wk, wflags, _, _ = osk.sk_flag(x[sl], M, N, 1.0, lo, hi)
        assert np.array_equal(y1[sl], wy), r0
        assert nan_equal(k1[sl], wk), r0
        nflag += int(wflags.sum())
    assert 0.02 < nflag / (x.shape[0] * 512) < 0.06


@pytest.mark.gpu
def test_workspace_protocol():
    rng = np.random.default_rng(9)
    M, N = 64, 2
    x = power(rng, (3, 4, 5000), np.uint16, scale=1000.)
    d_x = bf.asarray(x, space='cuda')
    nwin = sk_nwindow(5000, M)
    plan = SkFlag()
    plan.init(M, N)
    d_a, d_b = bf.zeros(x.shape, 'u16', 'cuda'), bf.zeros(x.shape, 'u16', 'cuda')
    k_a, k_b = bf.zeros((3, 4, nwin), 'f32', 'cuda'), bf.zeros((3, 4, nwin), 'f32', 'cuda')
    size = plan.get_workspace_size(d_x, d_a, k_a)              # (NULL, &size): query only
    assert size >= 3 * 4 * nwin * 9
    bf.device.stream_synchronize()
    assert np.all(host(d_a) == 0) and np.all(host(k_a) == 0)
    plan.execute(d_x, d_a, k_a)                                # (NULL, NULL): library-managed
    ws = bf.empty((size,), dtype='u8', space='cuda')
    plan.execute_workspace(d_x, d_b, ws.ctypes.data, size, k_b)   # (ptr, &size): caller's memory
    bf.device.stream_synchronize()
    a, b = host(d_a), host(d_b)
    assert np.array_equal(a, b) and np.array_equal(host(k_a).view(np.uint32), host(k_b).view(np.uint32))
    check_exact(x, a, host(k_a), M, N, 1.0, plan.lo, plan.hi)
    small = _bf.BFsize(size - 1)
    st = _bf.bfSkFlagExecute(plan.obj, d_x.as_BFarray(), d_b.as_BFarray(), None,
                             ctypes.c_void_p(ws.ctypes.data), ctypes.byref(small))
    assert st == _bf.BF_STATUS_INSUFFICIENT_STORAGE
    st = _bf.bfSkFlagExecute(plan.obj, d_x.as_BFarray(), d_b.as_BFarray(), None,
                             ctypes.c_void_p(ws.ctypes.data), None)
    assert st == _bf.BF_STATUS_INVALID_ARGUMENT


def status(plan, x, y, k=None):
    return _bf.bfSkFlagExecute(plan.obj if plan is not None else None, x.as_BFarray() if x is not None else None,
                               y.as_BFarray() if y is not None else None,
                               k.as_BFarray() if k is not None else None, None, None)


def fake(arr, shape, strides):
    """A BFarray on arr's memory with a shape far larger than the memory: only
    for calls that must refuse it before touching any data."""
    a = arr.as_BFarray()
    a.ndim = len(shape)
    for i, (n, s) in enumerate(zip(shape, strides)):
        a.shape[i], a.strides[i] = n, s
    return a


@pytest.mark.gpu
def test_error_statuses():
    M = 64
    plan = SkFlag()
    d_x = bf.zeros((2, 3, 1000), 'u8', 'cuda')
    d_y = bf.zeros((2, 3, 1000), 'u8', 'cuda')
    nwin = sk_nwindow(1000, M)
    d_k = bf.zeros((2, 3, nwin), 'f32', 'cuda')
    S = _bf
    assert status(plan, d_x, d_y) == S.BF_STATUS_INVALID_STATE
    plan.init(M, 1)
    assert status(plan, d_x, d_y) == S.BF_STATUS_SUCCESS
    assert status(plan, d_x, d_y, d_k) == S.BF_STATUS_SUCCESS
    assert status(None, d_x, d_y) == S.BF_STATUS_INVALID_HANDLE
    assert status(plan, None, d_y) == S.BF_STATUS_INVALID_POINTER
    assert status(plan, d_x, None) == S.BF_STATUS_INVALID_POINTER
    sys_x = bf.zeros((2, 3, 1000), 'u8')
    assert status(plan, sys_x, d_y) == S.BF_STATUS_UNSUPPORTED_SPACE
    assert status(plan, d_x, sys_x) == S.BF_STATUS_UNSUPPORTED_SPACE
    assert status(plan, d_x, d_y, bf.zeros((2, 3, nwin), 'f32')) == S.BF_STATUS_UNSUPPORTED_SPACE
    for dt in ('i8', 'i16', 'u32', 'f64', 'cf32'):
        assert status(plan, bf.zeros((2, 3, 1000), dt, 'cuda'), bf.zeros((2, 3, 1000), dt, 'cuda')) == \
            S.BF_STATUS_UNSUPPORTED_DTYPE, dt
    assert status(plan, d_x, bf.zeros((2, 3, 1000), 'u16', 'cuda')) == S.BF_STATUS_UNSUPPORTED_DTYPE
    assert status(plan, bf.zeros((2, 3, 1000), 'f32', 'cuda'), d_y) == S.BF_STATUS_UNSUPPORTED_DTYPE
    assert status(plan, d_x, d_y, bf.zeros((2, 3, nwin), 'f64', 'cuda')) == S.BF_STATUS_UNSUPPORTED_DTYPE
    for shape in ((3, 3, 1000), (2, 4, 1000), (2, 3, 999), (2, 3, 1000, 1), (6, 1000)):
        assert status(plan, d_x, bf.zeros(shape, 'u8', 'cuda')) == S.BF_STATUS_INVALID_SHAPE, shape
    for shape in ((2, 3, nwin + 1), (2, 3, nwin - 1), (3, 3, nwin), (2, 3), (2, 3, nwin, 1)):
        assert status(plan, d_x, d_y, bf.zeros(shape, 'f32', 'cuda')) == S.BF_STATUS_INVALID_SHAPE, shape
    wide = bf.zeros((2, 3, 2000), 'u8', 'cuda')
    assert status(plan, wide[:, :, ::2], d_y) == S.BF_STATUS_UNSUPPORTED_STRIDE
    assert status(plan, d_x, wide[:, :, ::2]) == S.BF_STATUS_UNSUPPORTED_STRIDE
    kwide = bf.zeros((2, 3, 2 * nwin), 'f32', 'cuda')
    assert status(plan, d_x, d_y, kwide[:, :, ::2]) == S.BF_STATUS_UNSUPPORTED_STRIDE
    # geometries past 32-bit rows / windows / samples, refused before any access
    big = [((1 << 31, 4), (0, 1)),                # rows > 2^31 - 1
           ((1 << 20, 1 << 12), (0, 1)),          # rows x windows = 2^31 with M = 2
           ((1 << 31,), (1,))]                    # ntime > 2^31 - 1 - M
    plan2 = SkFlag()
    plan2.init(2, 1)
    for shape, strides in big:
        a = fake(d_x, shape, strides)
        st = _bf.bfSkFlagExecute(plan2.obj, a, a, None, None, None)
        assert st == S.BF_STATUS_UNSUPPORTED_SHAPE, shape
        size = _bf.BFsize(0)
        st = _bf.bfSkFlagExecute(plan2.obj, a, a, None, None, ctypes.byref(size))
        assert st == S.BF_STATUS_UNSUPPORTED_SHAPE, shape
    bf.device.stream_synchronize()


@pytest.mark.gpu
def test_empty_inputs():
    plan = SkFlag()
    plan.init(16, 1)
    for shape in ((0, 100), (3, 0)):
        d = bf.zeros(shape, 'u8', 'cuda')
        k = bf.zeros(shape[:-1] + (sk_nwindow(shape[-1], 16),), 'f32', 'cuda')
        plan.execute(d, bf.zeros(shape, 'u8', 'cuda'), k)
    bf.device.stream_synchronize()


@pytest.mark.gpu
def test_kernel_path():
    from kernel_trace import device_kernels
    x = power(np.random.default_rng(10), (4, 3000), np.uint8)
    d_x = bf.asarray(x, space='cuda')
    d_y = bf.zeros(x.shape, 'u8', 'cuda')
    plan = SkFlag()
    plan.init(256, 4)
    plan.execute(d_x, d_y)                                     # workspace allocated outside the trace
    names = device_kernels(lambda: plan.execute(d_x, d_y))
    assert len(names) == 2
    assert 'sk_stats_kernel' in names[0] and 'sk_apply_kernel' in names[1]


# ------------------------------------------------------------------ pipeline
NCHAN, MD, GULP, NTIME = 256, 120, 4096, 3 * 4096 + 600
F0, DF, DT = 1200., 0.5, 1e-3
PULSES = ((0.2, 2000), (0.5, 4090), (0.9, 9000))            # the second straddles a gulp boundary
CARRIER = 40
BURST_CHANS = (100, 180)
BURSTS = ((4 * 256 + 154, 6 * 256 + 102), (20 * 256 + 154, 22 * 256 + 102), (40 * 256 + 154, 41 * 256 + 102))
IMPULSES = (3000, 6500, 11000, 12588)


def rfi_filterbank(seed=11):
    """u8 [time, freq]: Gamma(4, 8) noise, three dispersed two-sample pulses of
    32 (2 sigma) per channel, a constant carrier, two channels with bursts of
    +150 and broadband two-sample impulses of +200.  (Each search row is
    normalised by its own statistics, which an impulse dominates; a two-sample
    impulse keeps the zero-DM rows clearly ahead of the rows it smears into.)"""
    rng = np.random.default_rng(seed)
    x = rng.gamma(4., 8., size=(NCHAN, NTIME))
    f = F0 + DF * np.arange(NCHAN)
    rel = (f ** -2 - f[-1] ** -2) / (f[0] ** -2 - f[-1] ** -2)
    rows, pulse_mask = [], np.zeros(x.shape, bool)
    for frac, t0 in PULSES:
        tt = t0 + np.rint(rel * frac * (MD - 1)).astype(np.int64)
        for dt in (0, 1):
            x[np.arange(NCHAN), tt + dt] += 32.
            pulse_mask[np.arange(NCHAN), tt + dt] = True
        rows.append(int(np.rint(frac * (MD - 1))))
    rfi_mask = np.zeros(x.shape, bool)
    x[CARRIER] = 90.
    for c in BURST_CHANS:
        for a, b in BURSTS:
            x[c, a:b] += 150.
            rfi_mask[c, a:b] = True
    for t in IMPULSES:
        x[:, t:t + 2] += 200.
        rfi_mask[:, t:t + 2] = True
    x = np.clip(np.rint(x), 0, 255).astype(np.uint8)
    return np.ascontiguousarray(x.T), rows, pulse_mask, rfi_mask


def run_search(x, with_sk, widths, decim):
    from bifrost_b200 import blocks
    from bifrost_b200.pipeline import Pipeline
    hdr = {'_tensor': {'dtype': 'u8', 'shape': [-1, NCHAN], 'labels': ['time', 'freq'],
                       'scales': [[0, DT], [F0, DF]], 'units': ['s', 'MHz']},
           'name': 'fil', 'gulp_nframe': GULP}
    peaks, cleaned, heads = [], [], []
    with Pipeline() as p:
        src = blocks.array_source(x, hdr, gulp_nframe=GULP)
        b = blocks.copy(src, space='cuda')
        b = blocks.transpose(b, ['freq', 'time'])
        if with_sk:
            b = blocks.sk_flag(b, window=256, nacc=4)
            blocks.callback_sink(blocks.copy(b, space='system'), lambda q: heads.append(deepcopy(q.header)),
                                 lambda q: cleaned.append(np.array(q.data)))
        d = blocks.fdmt(b, max_delay=MD)
        s = blocks.pulse_search(d, widths=widths, decim=decim)
        blocks.callback_sink(blocks.copy(s, space='system'), None, lambda q: peaks.append(np.array(q.data)))
        p.run()
    return (np.concatenate(peaks, axis=1), np.concatenate(cleaned, axis=1) if with_sk else None,
            heads[0] if heads else None)


def brightest(got, decim, n=3):
    """The n brightest peaks, peaks within 1024 samples of a brighter one suppressed."""
    order = np.argsort(got[..., 0].ravel())[::-1]
    picks = []
    for i in order:
        r, j = divmod(int(i), got.shape[1])
        start = j * decim + int(got[r, j, 1])
        if all(abs(start - ps) > 1024 for _, ps, _ in picks):
            picks.append((r, start, int(got[r, j, 2])))
        if len(picks) == n:
            break
    return picks


@pytest.mark.gpu
def test_sk_flag_pipeline_removes_rfi():
    widths, decim, M = (1, 2, 4, 8, 16, 32), 256, 256
    x, rows, pulse_mask, rfi_mask = rfi_filterbank()
    xf = np.ascontiguousarray(x.T)                              # what sk_flag reads: [freq, time]
    # without sk_flag a zero-DM impulse is the brightest peak
    raw, _, _ = run_search(x, False, widths, decim)
    assert brightest(raw, decim, 1)[0][0] <= 2
    got, cleaned, head = run_search(x, True, widths, decim)
    assert head['sk_window'] == M and head['sk_nacc'] == 4
    assert head['_tensor']['dtype'] == 'u8' and head['_tensor']['labels'] == ['freq', 'time']
    assert cleaned.shape == xf.shape and cleaned.dtype == np.uint8
    # every output frame is the oracle on its gulp's span
    lo, hi = head['sk_thresholds']
    flags = []
    for g0 in range(0, NTIME, GULP):
        span = xf[:, g0:g0 + GULP]
        wy, _, wflags, _, _ = osk.sk_flag(span, M, 4, 1.0, lo, hi)
        assert np.array_equal(cleaned[:, g0:g0 + GULP], wy), g0
        flags.append(wflags)
    flags = np.concatenate(flags, axis=1)                       # windows never cross a gulp edge
    nwin = flags.shape[1]

    def windows(mask):
        pad = np.zeros((NCHAN, nwin * M - NTIME), bool)
        return np.concatenate([mask, pad], axis=1).reshape(NCHAN, nwin, M).any(axis=-1)
    assert np.all(flags[windows(rfi_mask)])
    assert np.all(flags[CARRIER])
    pw = windows(pulse_mask)
    assert flags[pw].sum() < 0.05 * pw.sum(), (flags[pw].sum(), pw.sum())
    # with it the three brightest peaks are the injected pulses
    picks = sorted(brightest(got, decim), key=lambda q: q[1])
    for (r, start, w), (frac, t0), row in zip(picks, PULSES, rows):
        assert abs(r - row) <= 2, (r, row)
        assert abs(start - t0) <= w + 1, (start, t0, w)
