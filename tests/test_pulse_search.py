"""bfPulseSearch*: boxcar S/N peak maps of a dispersion bank.

CPU: the oracle (oracle/pulse_search.py) against closed forms and a brute-force
restatement, and the block's output header.  GPU: bfPulseSearchExecute against
the oracle on strided / batched / edge-case banks, its statuses and workspace
protocol, bit-for-bit repeatability, the kernel path, and an int8 filterbank
through copy -> transpose -> fdmt -> pulse_search."""
import ctypes
import os
import sys
from copy import deepcopy

import numpy as np
import pytest

import bifrost_b200 as bf
from bifrost_b200.libbifrost import _bf
from bifrost_b200.blocks.pulse_search import pulse_search_header, PEAK_FIELDS
from bifrost_b200.pulse_search import PulseSearch, output_nblock
from oracle import pulse_search as ops

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

POW2 = (1, 2, 4, 8, 16, 32, 64, 128, 256)


# ------------------------------------------------------------------ oracle (CPU)
def tophat_snr(w, n):
    """Closed-form S/N at the peak of a width-w top-hat fully inside n starts,
    searched with width w: b = A * overlap, sum b = A w^2,
    sum b^2 = A^2 (w^2 + 2 sum_{k<w} k^2)."""
    s1 = w * w
    s2 = w * w + (w - 1) * w * (2 * w - 1) / 3
    mu = s1 / n
    return (w - mu) / np.sqrt(s2 / n - mu * mu)


@pytest.mark.parametrize('w,amp,base', [(1, 5.0, 0.0), (4, 3.0, 0.0), (16, 2.5, 7.0), (37, 1.0, -3.25)])
def test_oracle_tophat_closed_form(w, amp, base):
    ntime, p = 1000, 400
    x = np.full((1, ntime), base, np.float32)
    x[0, p:p + w] += amp
    nout = ntime - w + 1
    out, best = ops.pulse_search(x, [w], nout)
    assert out.shape == (1, 1, 3)
    np.testing.assert_allclose(best[0, 0], tophat_snr(w, nout), rtol=1e-12)
    assert out[0, 0, 1] == p and out[0, 0, 2] == w


def test_oracle_constant_rows_give_zero():
    x = np.empty((3, 500), np.float32)
    x[0], x[1], x[2] = 0., 3.7, -1e6
    out, best = ops.pulse_search(x, [2, 3, 9], 64)
    assert np.all(best == 0)
    assert np.all(out[..., 0] == 0) and np.all(out[..., 1] == 0) and np.all(out[..., 2] == 2)


def test_oracle_tie_breaking():
    # two equal pulses in one block: the first start wins
    x = np.zeros((1, 300), np.float32)
    x[0, 50] = x[0, 90] = 1.
    out, _ = ops.pulse_search(x, [1], 300)
    assert out[0, 0, 1] == 50 and out[0, 0, 2] == 1
    # all widths tie (s = 0 everywhere): the first width
    out, _ = ops.pulse_search(np.ones((1, 300), np.float32), [3, 5, 7], 100)
    assert np.all(out[0, :, 2] == 3) and np.all(out[0, :, 1] == 0)


def brute_force(x, widths, decim):
    ntime = x.shape[-1]
    W = max(widths)
    nout = ntime - W + 1
    nblk = -(-nout // decim)
    out = np.zeros(x.shape[:-1] + (nblk, 3))
    for r in np.ndindex(*x.shape[:-1]):
        row = x[r].astype(np.float64)
        b = [[sum(row[t + k] for k in range(w)) for t in range(nout)] for w in widths]
        mu = [sum(bw) / nout for bw in b]
        sd = [np.sqrt(sum((v - m) ** 2 for v in bw) / nout) for bw, m in zip(b, mu)]
        for j in range(nblk):
            best = None
            for wi, w in enumerate(widths):
                tw = None
                for t in range(j * decim, min((j + 1) * decim, nout)):
                    if tw is None or b[wi][t] > b[wi][tw]:
                        tw = t
                s = (b[wi][tw] - mu[wi]) / sd[wi] if sd[wi] > 0 else 0.
                if best is None or s > best[0]:
                    best = (s, tw - j * decim, w)
            out[r + (j,)] = best
    return out


@pytest.mark.parametrize('seed', range(4))
def test_oracle_equals_brute_force(seed):
    rng = np.random.default_rng(seed)
    nw = int(rng.integers(1, 5))
    widths = sorted(rng.choice(np.arange(1, 20), size=nw, replace=False).tolist())
    ntime = int(rng.integers(max(widths), 90))
    decim = int(rng.integers(1, 40))
    x = rng.integers(-4, 5, size=(2, 3, ntime)).astype(np.float32)
    out, _ = ops.pulse_search(x, widths, decim)
    want = brute_force(x, widths, decim)
    np.testing.assert_allclose(out[..., 0], want[..., 0], rtol=1e-6, atol=1e-6)
    np.testing.assert_array_equal(out[..., 1:], want[..., 1:])


# ------------------------------------------------------------------ header (CPU)
def bank_header(ndm=794, gulp=4096, batch=()):
    return {'_tensor': {'dtype': 'f32', 'shape': list(batch) + [ndm, -1],
                        'labels': ['pol'] * len(batch) + ['dispersion', 'time'],
                        'scales': [None] * len(batch) + [[0., 0.126], [12.5, 6.4e-5]],
                        'units': [None] * len(batch) + ['pc cm^-3', 's']},
            'name': 'bank', 'gulp_nframe': gulp, 'max_dm': 100.}


def test_block_header():
    ihdr = bank_header(batch=(2,))
    keep = deepcopy(ihdr)
    ohdr = pulse_search_header(ihdr, POW2, 256)
    assert ihdr == keep
    t = ohdr['_tensor']
    assert t['dtype'] == 'f32'
    assert t['shape'] == [2, 794, -1, 3]
    assert t['labels'] == ['pol', 'dispersion', 'time', 'peak']
    assert t['units'] == [None, 'pc cm^-3', 's', None]
    assert t['scales'] == [None, [0., 0.126], [12.5, 6.4e-5 * 256], None]
    assert ohdr['boxcar_widths'] == list(POW2)
    assert ohdr['peak_fields'] == PEAK_FIELDS == ['snr', 'offset', 'width']
    assert ohdr['max_dm'] == 100.
    with pytest.raises(KeyError):
        pulse_search_header({'_tensor': dict(ihdr['_tensor'], shape=[2, -1, 4096])}, POW2, 256)
    with pytest.raises(TypeError):
        pulse_search_header({'_tensor': dict(ihdr['_tensor'], dtype='i8')}, POW2, 256)


def test_output_nblock():
    assert output_nblock(4096 + 255, POW2, 256) == 16
    assert output_nblock(4096 + 256, POW2, 256) == 17
    assert output_nblock(255, POW2, 256) == 0
    assert output_nblock(256, POW2, 256) == 1


@pytest.mark.parametrize('widths,decim', [((), 4), ((0, 2), 4), ((2, 2), 4), ((3, 2), 4),
                                          ((4097,), 4), (tuple(range(1, 34)), 4), ((1,), 0),
                                          ((1,), (1 << 24) + 1)])
def test_init_rejects_bad_arguments(widths, decim):
    plan = PulseSearch()
    with pytest.raises(RuntimeError, match='INVALID_ARGUMENT'):
        plan.init(widths, decim)


# ------------------------------------------------------------------ GPU
def run(d_x, widths, decim, out=None):
    lead = d_x.shape[:-1]
    nblk = output_nblock(d_x.shape[-1], widths, decim)
    d_o = out if out is not None else bf.zeros(lead + (nblk, 3), 'f32', 'cuda')
    plan = PulseSearch()
    plan.init(widths, decim)
    plan.execute(d_x, d_o)
    bf.device.stream_synchronize()
    return np.asarray(d_o.copy('system'))


def check(got, x, widths, decim, rows=None, chunk=32):
    """GPU output against the oracle: |ds| <= 1e-5 max(1, |s|), and the GPU's
    (start, width) must score within that tolerance of the oracle's best, so
    it is the oracle's choice unless the runner-up is a near-tie.  `rows`
    (flat row indices) restricts the check."""
    widths = list(widths)
    x2 = np.asarray(x).reshape(-1, x.shape[-1])
    g2 = got.reshape(-1, got.shape[-2], 3)
    idx = np.arange(x2.shape[0]) if rows is None else np.asarray(rows)
    for c0 in range(0, len(idx), chunk):
        sel = idx[c0:c0 + chunk]
        _, s = ops.snr(x2[sel], widths)                      # [r, nw, nout]
        nout = s.shape[-1]
        g = g2[sel]
        for j in range(g.shape[1]):
            lo, hi = j * decim, min((j + 1) * decim, nout)
            best = s[:, :, lo:hi].max(axis=(1, 2))
            tol = 1e-5 * np.maximum(1., np.abs(best))
            assert np.all(np.abs(g[:, j, 0] - best) <= tol), (j, g[:, j, 0], best)
            off = g[:, j, 1].astype(np.int64)
            assert np.all((off >= 0) & (off < hi - lo)), (j, off)
            wi = np.searchsorted(widths, g[:, j, 2].astype(np.int64))
            assert np.all(np.asarray(widths)[np.minimum(wi, len(widths) - 1)] == g[:, j, 2])
            at = s[np.arange(len(sel)), wi, lo + off]
            assert np.all(at >= best - tol), (j, at, best)


def noise_bank(rng, shape, pulses=3):
    """Correlated noise (a running mean, like FDMT rows) plus a few boxcars."""
    x = rng.normal(size=shape).astype(np.float32)
    x = (x + np.roll(x, 1, -1) + np.roll(x, 2, -1)).astype(np.float32)
    flat = x.reshape(-1, shape[-1])
    for _ in range(pulses):
        r = rng.integers(flat.shape[0])
        w = int(rng.integers(1, 40))
        t = int(rng.integers(0, shape[-1] - w))
        flat[r, t:t + w] += 4.
    return x


CASES = {
    'batch':          ((2, 3), 5, 3000, POW2[:7], 256),
    'nwidth1':        ((), 4, 2500, (7,), 100),
    'nwidth32':       ((), 3, 5000, tuple(range(1, 30)) + (64, 100, 300), 512),
    'npow2_widths':   ((2,), 3, 4000, (3, 5, 11, 50), 300),
    'W1_decim1':      ((), 3, 700, (1,), 1),
    'decim_ragged':   ((), 4, 6001, (1, 2, 4, 8, 16), 384),
    'nout_lt_decim':  ((), 4, 300, (1, 4, 16), 1024),
    'decim_huge':     ((), 2, 20000, (2, 8), 1 << 24),
    'decim_segments': ((), 3, 9000, (1, 3, 9, 27), 1000),
    'W4096':          ((), 2, 10000, (1, 64, 1000, 4096), 2048),
    'small_decim':    ((), 2, 2000, (1, 2, 5), 7),
}


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(CASES))
def test_matches_oracle(name):
    batch, ndm, ntime, widths, decim = CASES[name]
    rng = np.random.default_rng(sorted(CASES).index(name))
    x = noise_bank(rng, batch + (ndm, ntime))
    got = run(bf.asarray(x, space='cuda'), widths, decim)
    assert got.shape == batch + (ndm, output_nblock(ntime, widths, decim), 3)
    check(got, x, widths, decim)


@pytest.mark.gpu
def test_row_pitch_and_unaligned_base():
    rng = np.random.default_rng(5)
    ndm, ntime, widths, decim = 6, 3000, (1, 2, 4, 8, 16, 32), 256
    big = noise_bank(rng, (2, ndm + 1, ntime + 37))
    d_big = bf.asarray(big, space='cuda')
    view = d_big[:, 1:, 1:1 + ntime]                      # row pitch ntime + 37, base + 1 element
    nblk = output_nblock(ntime, widths, decim)
    d_obig = bf.zeros((2, ndm, nblk + 3, 3), 'f32', 'cuda')
    oview = d_obig[:, :, 1:1 + nblk]
    plan = PulseSearch()
    plan.init(widths, decim)
    plan.execute(view, oview)
    bf.device.stream_synchronize()
    full = np.asarray(d_obig.copy('system'))
    check(full[:, :, 1:1 + nblk], big[:, 1:, 1:1 + ntime], widths, decim)
    assert np.all(full[:, :, 0] == 0) and np.all(full[:, :, 1 + nblk:] == 0)


@pytest.mark.gpu
def test_large_offset_leaves_snr_unchanged():
    rng = np.random.default_rng(6)
    widths, decim = POW2[:8], 256
    x = np.rint(noise_bank(rng, (8, 6000)) * 8).astype(np.float32)   # integers: x + 1e6 is exact
    got = run(bf.asarray(x + np.float32(1e6), space='cuda'), widths, decim)
    check(got, x, widths, decim)


@pytest.mark.gpu
def test_nan_row_leaves_other_rows_alone():
    rng = np.random.default_rng(7)
    widths, decim = (1, 4, 16), 128
    x = noise_bank(rng, (6, 3000))
    x[2, 1700] = np.nan
    x[4, 10] = np.inf
    got = run(bf.asarray(x, space='cuda'), widths, decim)
    check(got, x, widths, decim, rows=[0, 1, 3, 5])


@pytest.mark.gpu
def test_constant_rows():
    x = np.empty((3, 2000), np.float32)
    x[0], x[1], x[2] = 0., 3.7, -1e6
    got = run(bf.asarray(x, space='cuda'), (2, 3, 9), 256)
    assert np.all(got[..., 0] == 0) and np.all(got[..., 1] == 0) and np.all(got[..., 2] == 2)


@pytest.mark.gpu
def test_config2_shape_and_repeatability():
    rng = np.random.default_rng(8)
    ndm, ntime = 794, 131072
    x = rng.normal(size=(ndm, ntime)).astype(np.float32)
    for r, t, w in ((150, 20000, 1), (397, 65000, 12), (700, 100000, 100)):
        x[r, t:t + w] += 20. / np.sqrt(w)
    d_x = bf.asarray(x, space='cuda')
    a = run(d_x, POW2, 256)
    b = run(d_x, POW2, 256)
    assert a.shape == (ndm, 512, 3)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    check(a, x, POW2, 256, rows=np.r_[0:32, 140:160, 390:400, 690:710, 762:794], chunk=16)
    # the three injected pulses are the three brightest peaks
    top = np.argsort(a[..., 0].ravel())[::-1][:3]
    found = sorted((int(i // 512), int(i % 512)) for i in top)
    assert found == [(150, 20000 // 256), (397, 65000 // 256), (700, 100000 // 256)]


@pytest.mark.gpu
def test_workspace_protocol():
    rng = np.random.default_rng(9)
    widths, decim = (1, 2, 4, 8, 16), 200
    x = noise_bank(rng, (3, 4, 5000))
    d_x = bf.asarray(x, space='cuda')
    nblk = output_nblock(5000, widths, decim)
    plan = PulseSearch()
    plan.init(widths, decim)
    d_a = bf.zeros((3, 4, nblk, 3), 'f32', 'cuda')
    d_b = bf.zeros((3, 4, nblk, 3), 'f32', 'cuda')
    size = plan.get_workspace_size(d_x, d_a)                    # (NULL, &size): query only
    assert size > 0
    bf.device.stream_synchronize()
    assert np.all(np.asarray(d_a.copy('system')) == 0)
    plan.execute(d_x, d_a)                                      # (NULL, NULL): library-managed
    ws = bf.empty((size,), dtype='u8', space='cuda')
    plan.execute_workspace(d_x, d_b, ws.ctypes.data, size)     # (ptr, &size): caller's memory
    bf.device.stream_synchronize()
    a, b = np.asarray(d_a.copy('system')), np.asarray(d_b.copy('system'))
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    check(a, x, widths, decim)
    small = _bf.BFsize(size - 1)
    st = _bf.bfPulseSearchExecute(plan.obj, d_x.as_BFarray(), d_b.as_BFarray(),
                                  ctypes.c_void_p(ws.ctypes.data), ctypes.byref(small))
    assert st == _bf.BF_STATUS_INSUFFICIENT_STORAGE


def status(plan, x, o):
    return _bf.bfPulseSearchExecute(plan.obj, x.as_BFarray(), o.as_BFarray(), None, None)


@pytest.mark.gpu
def test_error_statuses():
    widths, decim = (1, 4, 16), 100
    plan = PulseSearch()
    d_x = bf.zeros((2, 3, 1000), 'f32', 'cuda')
    nblk = output_nblock(1000, widths, decim)
    d_o = bf.zeros((2, 3, nblk, 3), 'f32', 'cuda')
    assert status(plan, d_x, d_o) == _bf.BF_STATUS_INVALID_STATE
    plan.init(widths, decim)
    assert status(plan, d_x, d_o) == _bf.BF_STATUS_SUCCESS
    sys_x = bf.zeros((2, 3, 1000), 'f32')
    sys_o = bf.zeros((2, 3, nblk, 3), 'f32')
    assert status(plan, sys_x, d_o) == _bf.BF_STATUS_UNSUPPORTED_SPACE
    assert status(plan, d_x, sys_o) == _bf.BF_STATUS_UNSUPPORTED_SPACE
    assert status(plan, bf.zeros((2, 3, 1000), 'f64', 'cuda'), d_o) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    assert status(plan, bf.zeros((2, 3, 1000), 'i16', 'cuda'), d_o) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    assert status(plan, d_x, bf.zeros((2, 3, nblk, 3), 'i32', 'cuda')) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    for shape in ((3, 3, nblk, 3), (2, 4, nblk, 3), (2, 3, nblk + 1, 3), (2, 3, nblk - 1, 3),
                  (2, 3, nblk, 4), (2, 3, nblk)):
        assert status(plan, d_x, bf.zeros(shape, 'f32', 'cuda')) == _bf.BF_STATUS_INVALID_SHAPE, shape
    short = bf.zeros((2, 3, 15), 'f32', 'cuda')                 # ntime < W
    assert status(plan, short, bf.zeros((2, 3, 1, 3), 'f32', 'cuda')) == _bf.BF_STATUS_INVALID_SHAPE
    wide = bf.zeros((2, 3, 2000), 'f32', 'cuda')
    assert status(plan, wide[:, :, ::2], d_o) == _bf.BF_STATUS_UNSUPPORTED_STRIDE
    d_o2 = bf.zeros((2, 3, nblk, 6), 'f32', 'cuda')
    assert status(plan, d_x, d_o2[..., ::2]) == _bf.BF_STATUS_UNSUPPORTED_STRIDE
    with pytest.raises(RuntimeError, match='INVALID_ARGUMENT'):
        plan.init((4, 2), decim)
    assert _bf.bfPulseSearchExecute(None, d_x.as_BFarray(), d_o.as_BFarray(), None, None) == \
        _bf.BF_STATUS_INVALID_HANDLE
    bf.device.stream_synchronize()


@pytest.mark.gpu
def test_kernel_path():
    from kernel_trace import device_kernels
    x = noise_bank(np.random.default_rng(10), (4, 3000))
    d_x = bf.asarray(x, space='cuda')
    d_o = bf.zeros((4, output_nblock(3000, POW2, 256), 3), 'f32', 'cuda')
    plan = PulseSearch()
    plan.init(POW2, 256)
    plan.execute(d_x, d_o)                                      # workspace allocated outside the trace
    names = device_kernels(lambda: plan.execute(d_x, d_o))
    assert len(names) == 2
    assert 'pulse_search_scan_kernel' in names[0] and 'pulse_search_finish_kernel' in names[1]


# ------------------------------------------------------------------ pipeline
def filterbank(nchan, ntime, md, f0, df, pulses, seed):
    """round(N(0, 20)) int8 [time, freq] with dispersed one-sample pulses of
    100: (fraction of the max delay, arrival time at the top of the band)."""
    rng = np.random.default_rng(seed)
    x = np.clip(np.rint(rng.normal(0, 20, size=(nchan, ntime))), -127, 127).astype(np.int8)
    f = f0 + df * np.arange(nchan)
    rel = (f ** -2 - f[-1] ** -2) / (f[0] ** -2 - f[-1] ** -2)
    rows = []
    for frac, t0 in pulses:
        tt = t0 + np.rint(rel * frac * (md - 1)).astype(np.int64)
        x[np.arange(nchan), tt] = 100
        rows.append(int(np.rint(frac * (md - 1))))
    return np.ascontiguousarray(x.T), rows


@pytest.mark.gpu
def test_fdmt_pulse_search_pipeline():
    from bifrost_b200 import blocks
    from bifrost_b200.pipeline import Pipeline
    nchan, md, gulp, ntime = 256, 120, 4096, 3 * 4096 + 600
    f0, df, dt = 1200., 0.5, 1e-3
    widths, decim = (1, 2, 4, 8, 16, 32), 256
    pulses = ((0.2, 2000), (0.5, 4090), (0.9, 9000))          # the second straddles a gulp boundary
    x, rows = filterbank(nchan, ntime, md, f0, df, pulses, 11)
    hdr = {'_tensor': {'dtype': 'i8', 'shape': [-1, nchan], 'labels': ['time', 'freq'],
                       'scales': [[0, dt], [f0, df]], 'units': ['s', 'MHz']},
           'name': 'fil', 'gulp_nframe': gulp}
    banks, peaks, heads = [], [], []
    with Pipeline() as p:
        src = blocks.array_source(x, hdr, gulp_nframe=gulp)
        b = blocks.copy(src, space='cuda')
        b = blocks.transpose(b, ['freq', 'time'])
        d = blocks.fdmt(b, max_delay=md)
        blocks.callback_sink(blocks.copy(d, space='system'), None,
                             lambda s: banks.append(np.array(s.data)))
        s = blocks.pulse_search(d, widths=widths, decim=decim)
        blocks.callback_sink(blocks.copy(s, space='system'), lambda q: heads.append(deepcopy(q.header)),
                             lambda q: peaks.append(np.array(q.data)))
        p.run()
    bank = np.concatenate(banks, axis=1)
    got = np.concatenate(peaks, axis=1)
    t = heads[0]['_tensor']
    assert t['labels'] == ['dispersion', 'time', 'peak'] and t['shape'] == [md, -1, 3]
    assert heads[0]['boxcar_widths'] == list(widths)
    # every output frame is the oracle on the span its gulp searched
    ov = max(widths) - 1
    want_n, off = [], 0
    while True:
        span = bank[:, off:off + gulp + ov]
        if span.shape[1] <= ov:
            break
        nblk = output_nblock(span.shape[1], widths, decim)
        check(got[:, off // decim: off // decim + nblk], span, widths, decim)
        want_n.append(nblk)
        off += gulp
        if span.shape[1] < gulp + ov:
            break
    assert got.shape[1] == sum(want_n)
    # the three brightest peaks, one per pulse (peaks within 1024 samples suppressed)
    order = np.argsort(got[..., 0].ravel())[::-1]
    picks = []
    for i in order:
        r, j = divmod(int(i), got.shape[1])
        start = j * decim + int(got[r, j, 1])
        if all(abs(start - ps) > 1024 for _, ps, _ in picks):
            picks.append((r, start, int(got[r, j, 2])))
        if len(picks) == 3:
            break
    picks.sort(key=lambda q: q[1])
    for (r, start, w), (frac, t0), row in zip(picks, pulses, rows):
        assert abs(r - row) <= 2, (r, row)
        assert abs(start - t0) <= w + 1, (start, t0, w)
