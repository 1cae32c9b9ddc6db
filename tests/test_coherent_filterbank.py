"""bfCoherentDedispFilterbank: coherent dedispersion, fine channels, detection
and time integration in one pass (CoherentDedisp.filterbank and
coherent_dedisp(..., nfine=, detect=, nint=)).

CPU: the oracle (oracle/coherent_filterbank.py) against a per-fine-channel loop
with explicit DFTs, its nfine = 1 form against dedisperse -> detect -> sum,
the top-edge delay law of the fine channels for both sidebands, the block
header (scales, labels, coherent_nfine, fold_header's fine top edges) and its
refusals.  GPU: the op against the oracle for every dtype, mode, nfine, nint
and both kernel paths; bit for bit against bfCoherentDedispExecute -> bfDetect
-> bfReduce; views, repeatability, the workspace protocol, every status, the
kernel path, and GUPPI RAW -> coherent_dedisp(detect=) -> fold."""
import ctypes
import math
import os
import sys
from copy import deepcopy

import numpy as np
import pytest

import bifrost_b200 as bf
from bifrost_b200.libbifrost import _bf
from bifrost_b200.coherent_dedisp import CoherentDedisp, dispersion_overlap, default_nfft, filterbank_shape, KDM
from bifrost_b200.blocks.coherent_dedisp import coherent_filterbank_header, coherent_dedisp
from bifrost_b200.blocks.fold import fold_header
from oracle import coherent_dedisp as ocd
from oracle import coherent_filterbank as ocf

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

F0, DF = 1300.78125, 1.5625
MODES = ('scalar', 'stokes', 'stokes_i', 'coherence')
MODE_ID = {'scalar': 0, 'jones': 1, 'stokes': 2, 'stokes_i': 3, 'coherence': 4}


def cnoise(rng, shape):
    return rng.normal(size=shape) + 1j * rng.normal(size=shape)


# ------------------------------------------------------------------ oracle (CPU)
def brute_force(x, f0, df, dm, n, nfine, mode, nint):
    """Per fine channel and segment: explicit DFTs of the definition."""
    nchan, nb, ntime = x.shape
    m = ocd.overlap(nchan, f0, df, dm)
    q = nfine * nint
    step = q * ((n - m) // q)
    nf = n // nfine
    dff = df / nfine
    kk = np.arange(n)
    fwd = np.exp(-2j * np.pi * np.outer(kk, kk) / n)
    qq = np.arange(nf)
    inv = np.exp(2j * np.pi * np.outer(qq, qq) / nf)
    z = np.zeros((nchan, nfine, nb, ntime // nfine), complex)
    for c in range(nchan):
        fc = f0 + c * df
        for j in range(nfine):
            top = f0 + (c * nfine + j) * dff - df / 2 + dff / 2 + abs(dff) / 2
            k = (n // 2 + j * nf + qq) % n
            nu = np.where(k < n // 2, k, k - n) / n * df
            phi = np.sign(df) * KDM * dm * 1e6 * (nu * (fc ** -2 - top ** -2) - nu * nu / (fc * fc * (fc + nu)))
            h = np.exp(2j * np.pi * (phi - np.rint(phi)))
            for b in range(nb):
                s = 0
                while s < ntime:
                    seg = np.zeros(n, complex)
                    part = x[c, b, s:s + n]
                    seg[:len(part)] = part
                    Y = (fwd @ seg)[k] * h / n
                    zj = inv @ Y
                    keep = min(step, ntime - s) // nfine
                    z[c, j, b, s // nfine:s // nfine + keep] = zj[:keep]
                    s += step
    d = ocf.detect(z, mode).reshape(nchan * nfine, -1, ntime // nfine)
    return d.reshape(d.shape[0], d.shape[1], -1, nint).sum(-1)


@pytest.mark.parametrize('mode', MODES)
def test_oracle_matches_brute_force(mode):
    rng = np.random.default_rng(1)
    for f0, df, dm, n, nfine, nint, ntime in ((400., 0.5, 0.3, 256, 1, 2, 800),
                                              (1300.78125, -1.5625, 2., 512, 2, 3, 1200),
                                              (800., 1.5625, 1., 1024, 4, 1, 1600)):
        x = cnoise(rng, (2, 2, ntime))
        got = ocf.filterbank(x, f0, df, dm, n, nfine, mode, nint)
        want = brute_force(x, f0, df, dm, n, nfine, mode, nint)
        assert got.shape == want.shape == filterbank_shape(2, 2, ntime, nfine, mode, nint)
        assert np.abs(got - want).max() <= 1e-9 * np.abs(want).max(), (mode, n, nfine)


@pytest.mark.parametrize('mode', MODES)
def test_oracle_nfine1_is_dedisperse_detect_reduce(mode):
    rng = np.random.default_rng(2)
    n, dm = 1024, 5.
    m = ocd.overlap(3, F0, DF, dm)
    nint = next(d for d in range(2, n - m + 1) if (n - m) % d == 0)
    x = cnoise(rng, (3, 2, nint * 700))
    y = ocd.dedisperse(x, F0, DF, dm, n)
    d = ocf.detect(y, mode)
    want = d.reshape(d.shape[0], d.shape[1], -1, nint).sum(-1)
    got = ocf.filterbank(x, F0, DF, dm, n, 1, mode, nint)
    assert np.abs(got - want).max() <= 1e-10 * np.abs(want).max()


@pytest.mark.parametrize('df', [1.5625, -1.5625])
def test_fine_channels_peak_at_their_top_edge_delay(df):
    """An impulse dispersed with disperse comes out of every fine channel at
    that fine channel's own top-edge delay, D DM (f_top,j^-2 - f_top^-2)
    coarse samples after its position."""
    n, dm, t0, nfine = 8192, 100., 3000, 8
    ntime = 4 * n
    x = np.zeros((1, 1, ntime), complex)
    x[0, 0, t0] = 1.0
    y = ocd.disperse(x, F0, df, dm)
    z = ocf.fine_channels(y, F0, df, dm, n, nfine)[0, :, 0]           # [nfine, ntime / nfine]
    top = F0 + abs(df) / 2
    delays = []
    for j in range(nfine):
        topj = ocf.fine_top(F0, df, nfine, j)
        tau = KDM * dm * (topj ** -2 - top ** -2) * abs(df) * 1e6     # coarse samples
        p = np.abs(z[j]) ** 2
        peak = int(np.argmax(p))
        assert abs(peak * nfine - (t0 + tau)) <= nfine, (j, peak * nfine, t0 + tau)
        assert p[peak] > 0.3 / nfine ** 2          # |z| <= 1 / nfine; the pulse falls between fine samples
        delays.append(tau)
    # the fine channel at the coarse top edge has no delay, the lowest the most
    jtop = nfine - 1 if df > 0 else 0
    assert delays[jtop] == pytest.approx(0.0, abs=1e-6)
    order = np.argsort(delays)
    assert order[0] == jtop and order[-1] == nfine - 1 - jtop


def voltage_header(dtype='ci8', nchan=4, f0=400.78125, df=1.5625, labels=('freq', 'pol', 'time')):
    tsamp = 1.0 / abs(df) / 1e6
    shape = [nchan, 2, -1] if len(labels) == 3 else [nchan, -1]
    scales = [[f0, df], None, [0.0, tsamp]] if len(labels) == 3 else [[f0, df], [0.0, tsamp]]
    units = ['MHz', None, 's'] if len(labels) == 3 else ['MHz', 's']
    return {'_tensor': {'dtype': dtype, 'shape': shape, 'labels': list(labels), 'scales': scales, 'units': units},
            'name': 'v', 'gulp_nframe': 4096, 'refdm': 12.5, 'refdm_units': 'pc cm^-3'}


@pytest.mark.parametrize('df', [1.5625, -1.5625])
def test_filterbank_header(df):
    ihdr = voltage_header(df=df)
    keep = deepcopy(ihdr)
    ohdr, nfft, m, mode = coherent_filterbank_header(ihdr, 3.0, 4096, nfine=8, detect='stokes', nint=4)
    assert ihdr == keep
    assert (nfft, mode) == (4096, 'stokes') and m == dispersion_overlap(4, 400.78125, df, 3.0)
    t = ohdr['_tensor']
    assert t['dtype'] == 'f32' and t['labels'] == ['freq', 'pol', 'time'] and t['shape'] == [32, 4, -1]
    dff = df / 8
    assert t['scales'][0] == pytest.approx([400.78125 - df / 2 + dff / 2, dff], abs=1e-12)
    assert t['scales'][2] == pytest.approx([0.0, 32 / abs(df) / 1e6], rel=1e-12)
    assert ohdr['coherent_nfine'] == 8 and ohdr['coherent_dm'] == 3.0 and ohdr['coherent_nfft'] == 4096
    assert ohdr['gulp_nframe'] == 4096 // 32
    # fine centres tile the band: fine channel 0 of channel 0 starts at its coarse edge
    fine = t['scales'][0][0] + dff * np.arange(32)
    coarse = 400.78125 + df * np.arange(4)
    assert np.allclose(fine.reshape(4, 8).mean(1), coarse)
    # fold takes it unchanged: delays from the fine top edges
    _, delays, tsamp, _, _ = fold_header(ohdr, 64, 100.0)
    tops = fine + abs(dff) / 2
    want = KDM * 3.0 * (tops ** -2 - tops.max() ** -2)
    assert np.allclose(delays, want, rtol=1e-12, atol=1e-15) and tsamp == pytest.approx(32 / abs(df) / 1e6)
    for j in range(8):
        assert tops[j] == pytest.approx(ocf.fine_top(400.78125, df, 8, j), abs=1e-12)
    # scalar / stokes_i / a 2-D stream
    o2 = coherent_filterbank_header(ihdr, 3.0, 4096, nfine=2, detect='stokes_i')[0]
    assert o2['_tensor']['shape'] == [8, 1, -1] and o2['gulp_nframe'] == 2048
    assert o2['_tensor']['scales'][2][1] == pytest.approx(2 / abs(df) / 1e6)
    o3, _, _, m3 = coherent_filterbank_header(voltage_header(df=df, labels=('freq', 'time')), 3.0, 1024,
                                              nfine=4, detect='stokes')
    assert m3 == 'scalar' and o3['_tensor']['shape'] == [16, -1] and o3['_tensor']['dtype'] == 'f32'
    assert coherent_filterbank_header(ihdr, 3.0, 1024, detect='scalar')[0]['_tensor']['shape'] == [4, 2, -1]


def test_filterbank_rejections():
    ihdr = voltage_header()
    with pytest.raises(ValueError):                       # nfine / nint without detect
        coherent_dedisp(None, 3.0, nfine=2)
    with pytest.raises(ValueError):
        coherent_dedisp(None, 3.0, nint=4)
    with pytest.raises(ValueError):                       # nfine not a power of two
        coherent_filterbank_header(ihdr, 3.0, 4096, nfine=3, detect='stokes_i')
    with pytest.raises(ValueError):                       # N / nfine < 256
        coherent_filterbank_header(ihdr, 3.0, 1024, nfine=8, detect='stokes_i')
    with pytest.raises(ValueError):                       # jones has no power form
        coherent_filterbank_header(ihdr, 3.0, 1024, detect='jones')
    with pytest.raises(ValueError):
        coherent_filterbank_header(ihdr, 3.0, 1024, nint=0, detect='stokes_i')
    with pytest.raises(ValueError):
        filterbank_shape(4, 2, 1000, 16, 'stokes_i', 1)
    assert filterbank_shape(4, 3, 1024, 4, 'scalar', 2) == (16, 3, 128)
    assert filterbank_shape(4, 2, 1024, 1, 'coherence', 8) == (4, 4, 128)


# ------------------------------------------------------------------ GPU
def host(d):
    return np.asarray(d.copy('system'))


def make_input(rng, dtype, shape):
    """(host array for bf.asarray, complex128 values)."""
    if dtype == 'cf32':
        x = (rng.normal(size=shape) + 1j * rng.normal(size=shape)).astype(np.complex64) * 10
        return x, x.astype(np.complex128)
    if dtype == 'ci4':
        re = rng.integers(-8, 8, size=shape)
        im = rng.integers(-8, 8, size=shape)
        raw = (((re & 0xF) << 4) | (im & 0xF)).astype(np.uint8)
        return bf.ndarray(raw.view(bf.DataType('ci4').as_numpy_dtype()), dtype='ci4'), re + 1j * im
    lim = 127 if dtype == 'ci8' else 30000
    x = np.empty(shape, dtype=bf.DataType(dtype).as_numpy_dtype())
    x['re'] = rng.integers(-lim, lim + 1, size=shape)
    x['im'] = rng.integers(-lim, lim + 1, size=shape)
    return x, x['re'].astype(np.float64) + 1j * x['im'].astype(np.float64)


def check_rows(got, want, tol=2e-5):
    got = got.reshape(-1, got.shape[-1]).astype(np.float64)
    want = want.reshape(-1, want.shape[-1])
    assert got.shape == want.shape
    for r in range(got.shape[0]):
        peak = np.abs(want[r]).max()
        err = np.abs(got[r] - want[r]).max()
        assert err <= tol * peak, (r, err, peak)


def run_fb(d_x, f0, df, dm, n, nfine, mode, nint):
    plan = CoherentDedisp()
    plan.init(d_x.shape[0], f0, df, dm, n)
    d_o = bf.zeros(filterbank_shape(*d_x.shape, nfine, mode, nint), 'f32', 'cuda')
    plan.filterbank(d_x, d_o, nfine, mode, nint)
    bf.device.stream_synchronize()
    return host(d_o), plan


FB_CASES = {
    # N: (f0, df, dm, ntime)
    256:   (400.78125, 1.5625, 0.05, 64 * 50),
    1024:  (1350., -1.5625, 5., 64 * 150),
    4096:  (F0, DF, 100., 64 * 320),
    8192:  (F0, DF, 200., 64 * 500),
    65536: (F0, DF, 1000., 64 * 2200),
}


@pytest.mark.gpu
@pytest.mark.parametrize('nint', [1, 4])
@pytest.mark.parametrize('nfine', [1, 2, 16])
@pytest.mark.parametrize('n', sorted(FB_CASES))
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('dtype', ['ci4', 'ci8', 'ci16', 'cf32'])
def test_matches_oracle(dtype, mode, n, nfine, nint):
    if n // nfine < 256:
        pytest.skip("N / nfine < 256 is refused")
    f0, df, dm, ntime = FB_CASES[n]
    rng = np.random.default_rng(abs(hash((dtype, mode, n, nfine, nint))) % (1 << 31))
    x, xc = make_input(rng, dtype, (2, 2, ntime))
    got, _ = run_fb(bf.asarray(x, space='cuda'), f0, df, dm, n, nfine, mode, nint)
    check_rows(got, ocf.filterbank(xc, f0, df, dm, n, nfine, mode, nint))


def compose(plan, d_x, mode, nint):
    """bfCoherentDedispExecute -> bfDetect -> bfReduce."""
    nchan, nb, ntime = d_x.shape
    d_y = bf.zeros(d_x.shape, 'cf32', 'cuda')
    plan.execute(d_x, d_y)
    nprod = filterbank_shape(nchan, nb, ntime, 1, mode, 1)[1]
    d_d = bf.zeros((nchan, nprod, ntime), 'f32', 'cuda')
    if mode == 'scalar':
        bf.detect(d_y, d_d, 'scalar')
    else:
        bf.detect(d_y, d_d, mode, 1)
    if nint == 1:
        return host(d_d)
    d_r = bf.zeros((nchan, nprod, ntime // nint), 'f32', 'cuda')
    bf.reduce(d_d, d_r, 'sum')
    return host(d_r)


@pytest.mark.gpu
@pytest.mark.parametrize('n', [1024, 8192])
@pytest.mark.parametrize('mode', MODES)
def test_bit_exact_against_composition(mode, n):
    """nfine = 1 with S = L: the three calls' bits."""
    f0, df, dm = 1350., -1.5625, 20.
    rng = np.random.default_rng(11)
    plan = CoherentDedisp()
    plan.init(3, f0, df, dm, n)
    L = n - plan.overlap
    nints = [1] + [d for d in range(2, 33) if L % d == 0][:1]
    for dtype in ('ci8', 'cf32'):
        for nint in nints:
            ntime = nint * (3 * L // nint + 5)
            x, _ = make_input(rng, dtype, (3, 2, ntime))
            d_x = bf.asarray(x, space='cuda')
            want = compose(plan, d_x, mode, nint)
            d_o = bf.zeros(filterbank_shape(3, 2, ntime, 1, mode, nint), 'f32', 'cuda')
            plan.filterbank(d_x, d_o, 1, mode, nint)
            bf.device.stream_synchronize()
            got = host(d_o)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (dtype, nint)


@pytest.mark.gpu
@pytest.mark.parametrize('n,nfine', [(1024, 2), (2048, 8), (16384, 4)])
def test_strided_offset_views_and_negative_df(n, nfine):
    rng = np.random.default_rng(5)
    f0, df, dm, nint, mode = 1380., -1.5625, 20., 2, 'coherence'
    ntime = 12000
    x, xc = make_input(rng, 'ci8', (6, 3, ntime + 1))
    d_big = bf.asarray(x, space='cuda')
    d_x = d_big[::2, 1:, 1:]                       # channel stride 2 rows, pol offset, base + 1 sample
    want = ocf.filterbank(xc[::2, 1:, 1:], f0, df, dm, n, nfine, mode, nint)
    plan = CoherentDedisp()
    plan.init(3, f0, df, dm, n)
    shape = filterbank_shape(3, 2, ntime, nfine, mode, nint)
    d_out = bf.zeros((shape[0], shape[1], 2, shape[2] * 2), 'f32', 'cuda')
    d_o = d_out[:, :, 1, ::2]                      # strided rows and a time stride of 8 bytes
    plan.filterbank(d_x, d_o, nfine, mode, nint)
    bf.device.stream_synchronize()
    got = host(d_out)
    check_rows(np.ascontiguousarray(got[:, :, 1, ::2]), want)
    assert np.all(got[:, :, 0, :] == 0) and np.all(got[:, :, 1, 1::2] == 0)


@pytest.mark.gpu
@pytest.mark.parametrize('n', [2048, 16384])
def test_repeatable_and_workspace_protocol(n):
    rng = np.random.default_rng(6)
    nfine, nint, mode = 4, 2, 'stokes'
    x, xc = make_input(rng, 'ci8', (4, 2, 40000))
    d_x = bf.asarray(x, space='cuda')
    plan = CoherentDedisp()
    plan.init(4, F0, DF, 50., n)
    shape = filterbank_shape(4, 2, 40000, nfine, mode, nint)
    d_a, d_b, d_c = (bf.zeros(shape, 'f32', 'cuda') for _ in range(3))
    size = plan.get_filterbank_workspace_size(d_x, d_a, nfine, mode, nint)   # query only
    bf.device.stream_synchronize()
    assert np.all(host(d_a) == 0)
    if n <= 4096:
        assert size < 8 * n                        # no N-sized buffer
    else:
        q = nfine * nint
        nseg = -(-40000 // (q * ((n - plan.overlap) // q)))
        assert size >= 8 * 8 * nseg * n
    plan.filterbank(d_x, d_a, nfine, mode, nint)
    plan.filterbank(d_x, d_b, nfine, mode, nint)
    ws = bf.empty((size,), dtype='u8', space='cuda')
    plan.filterbank_workspace(d_x, d_c, ws.ctypes.data, size, nfine, mode, nint)
    bf.device.stream_synchronize()
    a, b, c = host(d_a), host(d_b), host(d_c)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert np.array_equal(a.view(np.uint32), c.view(np.uint32))
    check_rows(a, ocf.filterbank(xc, F0, DF, 50., n, nfine, mode, nint))
    small = _bf.BFsize(size - 1)
    st = _bf.bfCoherentDedispFilterbank(plan.obj, d_x.as_BFarray(), nfine, 2, nint, d_b.as_BFarray(),
                                        ctypes.c_void_p(ws.ctypes.data), ctypes.byref(small))
    assert st == _bf.BF_STATUS_INSUFFICIENT_STORAGE
    st = _bf.bfCoherentDedispFilterbank(plan.obj, d_x.as_BFarray(), nfine, 2, nint, d_b.as_BFarray(),
                                        ctypes.c_void_p(ws.ctypes.data), None)
    assert st == _bf.BF_STATUS_INVALID_ARGUMENT


def status(plan, x, y, nfine=1, mode='stokes_i', nint=1):
    return _bf.bfCoherentDedispFilterbank(plan.obj if plan is not None else None,
                                          x.as_BFarray() if x is not None else None, nfine,
                                          MODE_ID.get(mode, mode), nint,
                                          y.as_BFarray() if y is not None else None, None, None)


@pytest.mark.gpu
def test_error_statuses():
    S = _bf
    plan = CoherentDedisp()
    d_x = bf.zeros((4, 2, 1024), 'ci8', 'cuda')
    d_y = bf.zeros((4, 1, 1024), 'f32', 'cuda')
    assert status(plan, d_x, d_y) == S.BF_STATUS_INVALID_STATE
    plan.init(4, F0, DF, 10., 1024)                # M = 93
    assert status(plan, d_x, d_y) == S.BF_STATUS_SUCCESS
    assert status(None, d_x, d_y) == S.BF_STATUS_INVALID_HANDLE
    assert status(plan, None, d_y) == S.BF_STATUS_INVALID_POINTER
    assert status(plan, d_x, None) == S.BF_STATUS_INVALID_POINTER
    assert status(plan, bf.zeros((4, 2, 1024), 'ci8'), d_y) == S.BF_STATUS_UNSUPPORTED_SPACE
    for dt in ('i8', 'f32', 'cf64', 'u8'):
        assert status(plan, bf.zeros((4, 2, 1024), dt, 'cuda'), d_y) == S.BF_STATUS_UNSUPPORTED_DTYPE, dt
    for dt in ('cf32', 'f64', 'u16'):
        assert status(plan, d_x, bf.zeros((4, 1, 1024), dt, 'cuda')) == S.BF_STATUS_UNSUPPORTED_DTYPE, dt
    assert status(plan, d_x, d_y, mode='jones') == S.BF_STATUS_UNSUPPORTED
    assert status(plan, d_x, d_y, mode=7) == S.BF_STATUS_UNSUPPORTED
    for nfine, nint in ((3, 1), (0, 1), (8, 1), (1, 0), (1, -2), (2, 512)):   # 1024 / 8 < 256; 1024 > N - M
        assert status(plan, d_x, bf.zeros((4, 1, 1024), 'f32', 'cuda'), nfine=nfine, nint=nint) == \
            S.BF_STATUS_INVALID_ARGUMENT, (nfine, nint)
    assert status(plan, bf.zeros((4, 2, 1004), 'ci8', 'cuda'), bf.zeros((16, 1, 125), 'f32', 'cuda'),
                  nfine=4, nint=2) == S.BF_STATUS_INVALID_SHAPE      # 1004 % 8 != 0
    assert status(plan, bf.zeros((4, 3, 1024), 'ci8', 'cuda'), d_y) == S.BF_STATUS_INVALID_SHAPE   # nb != 2
    for shape in ((4, 4, 1024), (4, 1, 512), (8, 1, 1024), (4, 1024), (4, 1, 1024, 1)):
        assert status(plan, d_x, bf.zeros(shape, 'f32', 'cuda')) == S.BF_STATUS_INVALID_SHAPE, shape
    assert status(plan, d_x, bf.zeros((8, 1, 256), 'f32', 'cuda'), nfine=2, nint=2) == S.BF_STATUS_SUCCESS
    assert status(plan, d_x, bf.zeros((4, 2, 1024), 'f32', 'cuda'), mode='scalar') == S.BF_STATUS_SUCCESS
    assert status(plan, d_x, bf.zeros((4, 4, 1024), 'f32', 'cuda'), mode='coherence') == S.BF_STATUS_SUCCESS
    for shape in ((3, 2, 1024), (4, 1024)):        # nchan mismatch / no row axis
        assert status(plan, bf.zeros(shape, 'ci8', 'cuda'), d_y) == S.BF_STATUS_INVALID_SHAPE, shape
    wide = bf.zeros((4, 2, 2048), 'ci8', 'cuda')
    assert status(plan, wide[:, :, ::2], d_y) == S.BF_STATUS_UNSUPPORTED_STRIDE
    assert status(plan, bf.zeros((4, 2, 0), 'ci8', 'cuda'), bf.zeros((4, 1, 0), 'f32', 'cuda')) == \
        S.BF_STATUS_SUCCESS
    bf.device.stream_synchronize()


@pytest.mark.gpu
def test_kernel_path():
    from kernel_trace import device_kernels
    rng = np.random.default_rng(7)
    x, _ = make_input(rng, 'ci8', (4, 2, 32768))
    d_x = bf.asarray(x, space='cuda')
    for n, nfine in ((256, 1), (1024, 4), (4096, 16)):
        plan = CoherentDedisp()
        plan.init(4, F0, DF, 10., n)
        for mode in ('scalar', 'stokes'):
            d_o = bf.zeros(filterbank_shape(4, 2, 32768, nfine, mode, 2), 'f32', 'cuda')
            plan.filterbank(d_x, d_o, nfine, mode, 2)
            names = device_kernels(lambda: plan.filterbank(d_x, d_o, nfine, mode, 2))
            assert len(names) == 1 and 'coherent_filterbank_fused_kernel' in names[0], names
            assert plan.get_filterbank_workspace_size(d_x, d_o, nfine, mode, 2) < 8 * n
    for n, nfine in ((8192, 1), (65536, 16)):
        plan = CoherentDedisp()
        plan.init(4, F0, DF, 10., n)
        d_o = bf.zeros(filterbank_shape(4, 2, 32768, nfine, 'stokes_i', 4), 'f32', 'cuda')
        plan.filterbank(d_x, d_o, nfine, 'stokes_i', 4)    # workspace and bfFft tables outside the trace
        names = device_kernels(lambda: plan.filterbank(d_x, d_o, nfine, 'stokes_i', 4))
        assert 'coherent_dedisp_gather_kernel' in names[0], names
        assert 'coherent_filterbank_detect_kernel' in names[-1], names
        chirp = [i for i, s in enumerate(names) if 'coherent_dedisp_chirp_kernel' in s]
        assert len(chirp) == 1, names
        fwd, inv = names[1:chirp[0]], names[chirp[0] + 1:-1]
        assert fwd and inv and all('fft' in s for s in fwd + inv), names
        assert not any('fused' in s or 'keep' in s for s in names), names


# ------------------------------------------------------------------ pipeline
P_NCHAN, P_F0, P_DF, P_DM = 4, 400.78125, 1.5625, 1.0
P_NBLOCK, P_T0, P_PERIOD, P_AMP = 6, 700, 1500, 600.
P_NFINE, P_NINT, P_NBIN = 4, 2, 16


def pipeline_voltages(seed=17):
    """ci8 [block, chan, ntime, pol] of a GUPPI RAW file: noise of sigma 8 per
    component plus a pulse train (period P_PERIOD samples from P_T0), shifted
    per channel by its top-edge delay and then dispersed inside each channel."""
    m = dispersion_overlap(P_NCHAN, P_F0, P_DF, P_DM)
    nfft = default_nfft(m)
    q = P_NFINE * P_NINT
    step = q * ((nfft - m) // q)
    ntime = 2 * step
    total = P_NBLOCK * ntime
    rng = np.random.default_rng(seed)
    fc = P_F0 + P_DF * np.arange(P_NCHAN)
    tops = fc + P_DF / 2
    shift = np.rint(KDM * P_DM * (tops ** -2 - tops[-1] ** -2) * P_DF * 1e6).astype(int)
    imp = np.zeros((P_NCHAN, 2, total), complex)
    for c in range(P_NCHAN):
        for t in range(P_T0, total - 2 * m, P_PERIOD):
            imp[c, :, t + shift[c]] = P_AMP * np.array([1.0, 0.6 - 0.5j])
    v = ocd.disperse(imp, P_F0, P_DF, P_DM) + 8 * (rng.normal(size=imp.shape) + 1j * rng.normal(size=imp.shape))
    re = np.clip(np.rint(v.real), -127, 127).astype(np.int8)
    im = np.clip(np.rint(v.imag), -127, 127).astype(np.int8)
    data = np.stack([re, im], -1).reshape(P_NCHAN, 2, P_NBLOCK, ntime, 2).transpose(2, 0, 3, 1, 4)
    return np.ascontiguousarray(data), m, nfft, ntime


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


@pytest.mark.gpu
def test_guppi_filterbank_fold(tmp_path):
    from bifrost_b200 import blocks, views
    from bifrost_b200.pipeline import Pipeline
    data, m, nfft, ntime = pipeline_voltages()
    path = str(tmp_path / 'pulsar.raw')
    write_guppi(path, data)
    nu = 1.0 / (P_PERIOD / (P_DF * 1e6))
    power, profiles, heads = [], [], []
    with Pipeline() as p:
        b = blocks.read_guppi_raw([path])
        b = blocks.copy(b, space='cuda')
        b = blocks.transpose(b, ['freq', 'pol', 'time', 'fine_time'])
        b = views.merge_axes(b, 'time', 'fine_time')
        b = blocks.coherent_dedisp(b, P_DM, nfine=P_NFINE, detect='stokes_i', nint=P_NINT)
        blocks.callback_sink(blocks.copy(b, space='system'), lambda q: heads.append(deepcopy(q.header)),
                             lambda q: power.append(np.array(q.data)))
        f = blocks.fold(b, P_NBIN, nu)
        blocks.callback_sink(blocks.copy(f, space='system'), None, lambda q: profiles.append(np.array(q.data)))
        p.run()
    head = heads[0]
    q = P_NFINE * P_NINT
    assert head['coherent_nfine'] == P_NFINE and head['coherent_nfft'] == nfft
    assert head['_tensor']['labels'] == ['freq', 'pol', 'time'] and head['_tensor']['dtype'] == 'f32'
    got = np.concatenate(power, axis=-1)
    total = data.shape[0] * ntime
    ahead = -(-m // ntime) * ntime                  # whole GUPPI blocks (a multiple of q)
    assert got.shape == (P_NCHAN * P_NFINE, 1, (total - ahead) // q)
    # the gulp (one GUPPI block) is a multiple of the segment step: the op on the whole stream
    x = np.ascontiguousarray(data.transpose(1, 3, 0, 2, 4).reshape(P_NCHAN, 2, total, 2))
    xs = np.empty((P_NCHAN, 2, total), dtype=bf.DataType('ci8').as_numpy_dtype())
    xs['re'], xs['im'] = x[..., 0], x[..., 1]
    whole, _ = run_fb(bf.asarray(xs, space='cuda'), P_F0, P_DF, P_DM, nfft, P_NFINE, 'stokes_i', P_NINT)
    assert np.array_equal(got.view(np.uint32), whole[..., :got.shape[-1]].view(np.uint32))
    # the pulse folds to its phase in every fine channel, from the header alone
    prof = np.sum(profiles, axis=0).reshape(P_NCHAN * P_NFINE, P_NBIN)
    want = int(math.floor((P_T0 / P_PERIOD % 1.0) * P_NBIN))
    for i in range(P_NCHAN * P_NFINE):
        peak = int(np.argmax(prof[i]))
        assert min((peak - want) % P_NBIN, (want - peak) % P_NBIN) <= 1, (i, peak, want)
        assert prof[i, peak] > 5 * np.median(prof[i]), (i, prof[i])
