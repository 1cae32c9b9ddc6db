"""Edges of bfLinAlgMatMul's integer kernels: the correlator (b^H.b and a.a^H
forms; corr_tc_kernel on the tensor cores, corr_simt_kernel otherwise) and the
ci8 a.b product (ab_tc_kernel).

Every correlator test asserts which kernel ran, read from the device activity
that torch.profiler records (it sees launches from libbifrost_b200.so too):
both kernels make one launch per call, so a silent fall-back to SIMT would
otherwise pass unnoticed.  Integer results are compared bit for bit with
oracle/linalg.py (exact integer sums, rounded once to fp32) over the full int8
range, -128 included; float inputs and time-chunked integrations within
1e-6 sqrt(|C_ii| |C_jj|) per element."""
import contextlib
import os

import numpy as np
import pytest

import bifrost_b200 as bf
from bifrost_b200.libbifrost import _bf
from bifrost_b200.linalg import LinAlg
from kernel_trace import device_kernels
from oracle import linalg as olinalg

pytestmark = pytest.mark.gpu

CI8 = bf.DataType('ci8').as_numpy_dtype()
CI16 = bf.DataType('ci16').as_numpy_dtype()


# ------------------------------------------------------------------ helpers
def corr_paths(names):
    """'tc' / 'simt' for each correlator kernel among `names`."""
    return ['tc' if 'corr_tc_kernel' in k else 'simt' for k in names if 'corr_tc_kernel' in k or 'corr_simt_kernel' in k]


@contextlib.contextmanager
def forced_simt(on=True):
    if on:
        os.environ['BFB_LINALG_SIMT'] = '1'
    try:
        yield
    finally:
        if on:
            del os.environ['BFB_LINALG_SIMT']


def correlate_dev(xv, c, alpha=1.0, beta=0.0, simt=False, aah=False):
    """c <- alpha xv^H.xv (or xv.xv^H) + beta c on the device.  Returns c on
    the host and the correlator kernels that ran."""
    la = LinAlg()
    reset = None
    if beta != 0:                                            # the result depends on c: restore it
        c0 = np.asarray(c.copy('system'))

        def reset():
            c[...] = c0
    with forced_simt(simt):
        names = device_kernels(lambda: la.matmul(alpha, xv if aah else None, None if aah else xv, beta, c),
                               reset=reset)
    return np.asarray(c.copy('system')), corr_paths(names)


def full_range_ci8(rng, shape):
    """Uniform over [-128, 127], with -128 forced into whole rows: every
    station of some time samples (real part) and every sample of station 0
    (both parts)."""
    x = np.empty(shape, dtype=CI8)
    x['re'] = rng.integers(-128, 128, size=shape)
    x['im'] = rng.integers(-128, 128, size=shape)
    x['re'][3::5] = -128
    x['re'][..., 0] = -128
    x['im'][..., 0] = -128
    return x


def as_complex(x):
    return x['re'].astype(np.float64) + 1j * x['im'].astype(np.float64)


def sentinel(shape):
    return (np.arange(int(np.prod(shape))).reshape(shape) % 7 + 0.5 - 3j).astype(np.complex64)


def assert_close_to_scale(got, want):
    """|got - want| <= 1e-6 sqrt(|C_ii| |C_jj|), element by element (lower triangle)."""
    d = np.abs(np.diagonal(want, axis1=-2, axis2=-1).real).astype(np.float64)
    tol = 1e-6 * np.sqrt(d[..., :, None] * d[..., None, :])
    il = np.tril_indices(want.shape[-1])
    err = np.abs(got.astype(np.complex128) - want)[..., il[0], il[1]]
    bound = tol[..., il[0], il[1]]
    assert (err <= bound).all(), "max err / bound = %g" % (err / np.maximum(bound, 1e-30)).max()


# ------------------------------------------------ tensor-core shape sweep
# n: T = ceil(2n / 128) row blocks of 1..8, 11 and 16 (odd and even: both
# operand-aliasing cases), n a multiple of 64 and not; n = 704 is 352 stands
# x 2 pols.  ntime: slab tails, multiples of the 3-stage ring, phase wrap.
SWEEP_N = [16, 24, 56, 64, 72, 120, 128, 136, 192, 200, 256, 264, 320, 384, 392, 448, 512, 704, 1024]
SWEEP_NTIME = [1, 8, 63, 64, 65, 191, 192, 193, 640]
# (n, ntime, nchan) of the sweep that do not reach the tensor cores: none.
# Every shape, including the ones smaller than one 64 x 128 B TMA box
# (n = 16, 24, 56; ntime < 64), takes corr_tc_kernel.
SWEEP_SIMT = set()


@pytest.mark.parametrize("n", SWEEP_N)
def test_tc_sweep_exact_and_bitwise_equal_to_simt(n):
    rng = np.random.default_rng(1000 + n)
    cases = [(ntime, nchan) for ntime in SWEEP_NTIME for nchan in (1, 3)]
    xs = [full_range_ci8(rng, (ntime, nchan, n)) for ntime, nchan in cases]
    d_xs = [bf.asarray(x, space='cuda') for x in xs]
    la = LinAlg()
    got = {}
    for simt in (False, True):
        d_cs = [bf.asarray(sentinel((nchan, n, n)), space='cuda') for _, nchan in cases]

        def run():
            for d_x, d_c in zip(d_xs, d_cs):
                la.matmul(1, None, d_x.transpose((1, 0, 2)), 0, d_c)
        with forced_simt(simt):
            paths = corr_paths(device_kernels(run))
        want_paths = ['simt' if simt or (n, ntime, nchan) in SWEEP_SIMT else 'tc' for ntime, nchan in cases]
        assert paths == want_paths, list(zip(cases, paths))
        got[simt] = [np.asarray(d_c.copy('system')) for d_c in d_cs]
        del d_cs
    for (ntime, nchan), x, tc, simt in zip(cases, xs, got[False], got[True]):
        want = olinalg.correlate(np.transpose(x, (1, 0, 2)), c=sentinel((nchan, n, n)))
        msg = str((n, ntime, nchan))
        np.testing.assert_array_equal(tc, want, err_msg=msg)          # incl. the untouched upper triangle
        np.testing.assert_array_equal(tc.view(np.uint32), simt.view(np.uint32), err_msg=msg)


# ------------------------------------------------------------ input views
@pytest.mark.parametrize("simt", [False, True])
def test_conjugated_input_view(simt):
    rng = np.random.default_rng(11)
    x = full_range_ci8(rng, (193, 3, 136))
    d_x = bf.asarray(x, space='cuda')
    c0 = sentinel((3, 136, 136))
    got, paths = correlate_dev(d_x.transpose((1, 0, 2)).conj(), bf.asarray(c0, space='cuda'), simt=simt)
    assert paths == ['simt' if simt else 'tc']
    want = olinalg.correlate(np.conj(np.transpose(as_complex(x), (1, 0, 2))), c=c0)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("simt", [False, True])
def test_strided_output_rows_and_batches(simt):
    """C as a view of a buffer padded in rows and between batch entries: the
    padding keeps its sentinel, the view gets the exact values."""
    rng = np.random.default_rng(12)
    nchan, ntime, n = 3, 130, 200
    x = full_range_ci8(rng, (ntime, nchan, n))
    big0 = sentinel((nchan, n + 5, n + 3))
    d_big = bf.asarray(big0, space='cuda')
    d_c = d_big[:, :n, :n]
    got, paths = correlate_dev(bf.asarray(x, space='cuda').transpose((1, 0, 2)), d_c, simt=simt)
    assert paths == ['simt' if simt else 'tc']
    want = big0.copy()
    want[:, :n, :n] = olinalg.correlate(np.transpose(x, (1, 0, 2)), c=big0[:, :n, :n])
    np.testing.assert_array_equal(np.asarray(d_big.copy('system')), want)


# -------------------------------------------------------- batch structure
def test_two_batch_dims_of_equal_size():
    rng = np.random.default_rng(13)
    x = full_range_ci8(rng, (100, 3, 3, 64))                 # [time, b1, b2, n]
    d_c = bf.zeros((3, 3, 64, 64), 'cf32', 'cuda')
    got, paths = correlate_dev(bf.asarray(x, space='cuda').transpose((1, 2, 0, 3)), d_c)
    assert paths == ['tc'] * 3                               # b2 in the grid, b1 looped
    np.testing.assert_array_equal(got, olinalg.correlate(np.transpose(x, (1, 2, 0, 3))))


def test_broadcast_kernel_batch_dim():
    """One input for every output batch entry (zero batch stride): TMA cannot
    describe it, so the SIMT kernel runs."""
    rng = np.random.default_rng(14)
    x = full_range_ci8(rng, (1, 70, 48))                     # [1, time, n]
    d_c = bf.zeros((4, 48, 48), 'cf32', 'cuda')
    got, paths = correlate_dev(bf.asarray(x, space='cuda'), d_c)
    assert paths == ['simt']
    np.testing.assert_array_equal(got, olinalg.correlate(np.broadcast_to(x, (4, 70, 48))))


def test_broadcast_outer_batch_dim():
    rng = np.random.default_rng(15)
    x = full_range_ci8(rng, (1, 3, 70, 48))                  # [1, chan, time, n]
    d_c = bf.zeros((2, 3, 48, 48), 'cf32', 'cuda')
    got, paths = correlate_dev(bf.asarray(x, space='cuda'), d_c)
    assert paths == ['tc', 'tc']
    np.testing.assert_array_equal(got, olinalg.correlate(np.broadcast_to(x, (2, 3, 70, 48))))


def test_outer_batch_stride_mixes_tc_and_simt():
    """Outer batch entries 8 bytes off a 16-byte boundary: entry 0 is aligned
    and takes the tensor cores, entry 1 cannot and takes SIMT, in one call."""
    import torch
    rng = np.random.default_rng(16)
    nouter, nchan, ntime, n = 2, 2, 96, 40
    block = ntime * nchan * n * 2                            # bytes of one [time, chan, n] entry
    s_outer = block + 8
    xs = [full_range_ci8(rng, (ntime, nchan, n)) for _ in range(nouter)]
    raw = np.zeros(s_outer * nouter, np.uint8)
    for o, x in enumerate(xs):
        raw[o * s_outer:o * s_outer + block] = x.view(np.uint8).ravel()
    buf = torch.from_numpy(raw).cuda()
    xv = bf.ndarray(space='cuda', shape=(nouter, nchan, ntime, n), dtype='ci8', buffer=buf.data_ptr(),
                    strides=(s_outer, 2 * n, 2 * n * nchan, 2))
    d_c = bf.zeros((nouter, nchan, n, n), 'cf32', 'cuda')
    got, paths = correlate_dev(xv, d_c)
    assert paths == ['tc', 'simt']
    want = olinalg.correlate(np.stack([np.transpose(x, (1, 0, 2)) for x in xs]))
    np.testing.assert_array_equal(got, want)


# --------------------------------------------------------- alpha and beta
@pytest.mark.parametrize("simt", [False, True])
def test_alpha_beta(simt):
    rng = np.random.default_rng(17)
    x = full_range_ci8(rng, (100, 2, 48))
    c0 = (rng.integers(-50, 50, size=(2, 48, 48)) + 1j * rng.integers(-50, 50, size=(2, 48, 48))).astype(np.complex64)
    got, paths = correlate_dev(bf.asarray(x, space='cuda').transpose((1, 0, 2)), bf.asarray(c0, space='cuda'),
                               alpha=0.5, beta=2.0, simt=simt)
    assert paths == ['simt' if simt else 'tc']
    np.testing.assert_array_equal(got, olinalg.correlate(np.transpose(x, (1, 0, 2)), c=c0, alpha=0.5, beta=2.0))


def test_aah_form_with_beta():
    """c = alpha a.a^H + beta c, i.e. u(t, i) = conj(a[i][t]): the SIMT kernel."""
    rng = np.random.default_rng(18)
    a = full_range_ci8(rng, (2, 24, 100))                    # [batch, n, ntime]
    c0 = (rng.integers(-50, 50, size=(2, 24, 24)) + 1j * rng.integers(-50, 50, size=(2, 24, 24))).astype(np.complex64)
    got, paths = correlate_dev(bf.asarray(a, space='cuda'), bf.asarray(c0, space='cuda'), alpha=0.5, beta=2.0,
                               aah=True)
    assert paths == ['simt']
    u = np.conj(np.swapaxes(as_complex(a), -1, -2))
    np.testing.assert_array_equal(got, olinalg.correlate(u, c=c0, alpha=0.5, beta=2.0))


# ------------------------------------------------------- non-int8 inputs
def test_ci16_at_full_scale():
    rng = np.random.default_rng(19)
    shape = (200, 2, 40)
    x = np.empty(shape, dtype=CI16)
    x['re'] = rng.choice([-32767, 32767], size=shape)
    x['im'] = rng.choice([-32767, 32767], size=shape)
    mix = rng.random(shape) < 0.3
    x['re'][mix] = rng.integers(-32767, 32768, size=int(mix.sum()))
    got, paths = correlate_dev(bf.asarray(x, space='cuda').transpose((1, 0, 2)), bf.zeros((2, 40, 40), 'cf32', 'cuda'))
    assert paths == ['simt']
    assert_close_to_scale(got, olinalg.correlate(np.transpose(as_complex(x), (1, 0, 2))))


def test_cf32_conjugated_and_batched():
    rng = np.random.default_rng(20)
    x = (rng.normal(size=(3, 200, 40)) + 1j * rng.normal(size=(3, 200, 40))).astype(np.complex64)
    got, paths = correlate_dev(bf.asarray(x, space='cuda').conj(), bf.zeros((3, 40, 40), 'cf32', 'cuda'))
    assert paths == ['simt']
    assert_close_to_scale(got, olinalg.correlate(np.conj(x.astype(np.complex128))))


# ------------------------------------------------------ long integrations
# Past 2^31 an int32 sum wraps: these lengths need the 64-bit epilogue
# combine and the time chunking of correlate().
def test_long_integration_full_scale_127():
    """ntime = 70000 of 127+127j: C = 70000 x 2 x 127^2 = 2258060000 > 2^31.
    One exact tensor-core pass; under BFB_LINALG_SIMT two SIMT chunks."""
    ntime, n = 70000, 16
    x = np.empty((ntime, 1, n), dtype=CI8)
    x['re'] = 127
    x['im'] = 127
    d_x = bf.asarray(x, space='cuda').transpose((1, 0, 2))
    want = olinalg.correlate(np.transpose(x, (1, 0, 2)))
    assert want[0, 0, 0].real == np.float32(2258060000)
    got, paths = correlate_dev(d_x, bf.zeros((1, n, n), 'cf32', 'cuda'))
    np.testing.assert_array_equal(got, want)
    assert paths == ['tc']
    got, paths = correlate_dev(d_x, bf.zeros((1, n, n), 'cf32', 'cuda'), simt=True)
    assert_close_to_scale(got, want)
    assert paths == ['simt', 'simt']                          # 65535 + 4465 samples
    check_autocorrelations(got)


def test_long_integration_minus_128():
    """ntime = 65536 of -128-128j: each Gram entry is 2^30, Re C = 2^31."""
    ntime, n = 65536, 16
    x = np.empty((ntime, 1, n), dtype=CI8)
    x['re'] = -128
    x['im'] = -128
    got, paths = correlate_dev(bf.asarray(x, space='cuda').transpose((1, 0, 2)), bf.zeros((1, n, n), 'cf32', 'cuda'))
    want = olinalg.correlate(np.transpose(x, (1, 0, 2)))
    assert want[0, 0, 0] == np.float32(2 ** 31)
    np.testing.assert_array_equal(got, want)
    assert paths == ['tc']
    check_autocorrelations(got)


def test_long_integration_chunked_on_the_tensor_cores():
    ntime, n = 300000, 16
    rng = np.random.default_rng(21)
    x = full_range_ci8(rng, (ntime, 1, n))
    c0 = sentinel((1, n, n))
    got, paths = correlate_dev(bf.asarray(x, space='cuda').transpose((1, 0, 2)), bf.asarray(c0, space='cuda'))
    want = olinalg.correlate(np.transpose(x, (1, 0, 2)), c=c0)
    assert_close_to_scale(got, want)
    assert paths == ['tc'] * 3                               # 131071 + 131071 + 37858 samples
    iu = np.triu_indices(n, 1)
    np.testing.assert_array_equal(got[:, iu[0], iu[1]], c0[:, iu[0], iu[1]])
    check_autocorrelations(got)


def check_autocorrelations(c):
    d = np.diagonal(c, axis1=-2, axis2=-1)
    assert (d.real > 0).all() and (d.imag == 0).all()


# ------------------------------------------- ci8 a.b on the tensor cores
def ab_gold(a, b, ca=False, cb=False):
    """Exact integer a.b (either operand conjugated), rounded once to cf32."""
    ar, ai = a['re'].astype(np.int64), a['im'].astype(np.int64)
    br, bi = b['re'].astype(np.int64), b['im'].astype(np.int64)
    sa, sb = (-1 if ca else 1), (-1 if cb else 1)
    re = ar @ br - (sa * ai) @ (sb * bi)
    im = ar @ (sb * bi) + (sa * ai) @ br
    return re.astype(np.float64).astype(np.float32) + 1j * im.astype(np.float64).astype(np.float32)


def ab_dev(la, a, b, ca=False, cb=False):
    da, db = bf.asarray(a, space='cuda'), bf.asarray(b, space='cuda')
    dc = bf.asarray(np.full(a.shape[:-1] + b.shape[-1:], 7 - 3j, np.complex64), space='cuda')
    names = device_kernels(lambda: la.matmul(1, da.conj() if ca else da, db.conj() if cb else db, 0, dc))
    assert any('ab_tc_kernel' in k for k in names), names
    return np.asarray(dc.copy('system'))


@pytest.mark.parametrize("m,n,k", [(1, 8, 1), (1, 8, 63), (5, 8, 64), (33, 200, 63), (64, 136, 64), (1, 8, 4096)])
def test_ab_minus_128_exact(m, n, k):
    rng = np.random.default_rng(m * 1000 + n + k)
    a, b = full_range_ci8(rng, (m, k)), full_range_ci8(rng, (k, n))
    a['re'][:, 1::3] = -128
    b['im'][::2] = -128
    la = LinAlg()
    for ca in (False, True):
        for cb in (False, True):
            np.testing.assert_array_equal(ab_dev(la, a, b, ca, cb), ab_gold(a, b, ca, cb), err_msg=str((ca, cb)))


def test_ab_cancellation_past_2_24_rounds_once():
    """K = 4096 with every part in [120, 127]: Gram terms pass 2^24 and cancel
    in Re = G00 - G11.  Converting each to fp32 before combining them (a
    model of that is checked to differ here) is not the correctly rounded
    exact sum; the kernel must be."""
    m, n, k = 4, 8, 4096
    rng = np.random.default_rng(22)
    a, b = np.empty((m, k), CI8), np.empty((k, n), CI8)
    for x in (a, b):
        x['re'] = rng.integers(120, 128, size=x.shape)
        x['im'] = rng.integers(120, 128, size=x.shape)
    ar, ai = a['re'].astype(np.int64), a['im'].astype(np.int64)
    br, bi = b['re'].astype(np.int64), b['im'].astype(np.int64)
    g00, g11, g01, g10 = ar @ br, ai @ bi, ar @ bi, ai @ br
    f = np.float32
    rounded_twice = (g00.astype(f) - g11.astype(f)) + 1j * (g01.astype(f) + g10.astype(f))
    gold = ab_gold(a, b)
    assert (rounded_twice != gold).any()
    got = ab_dev(LinAlg(), a, b)
    np.testing.assert_array_equal(got, gold)


def test_ab_long_reduction_past_int32():
    """K = 70000 of -128-128j: each Gram term is 70000 x 2^14 < 2^31, their
    sum (|Re| or |Im| = 2293760000, depending on the conjugation flags) is not."""
    m, n, k = 1, 8, 70000
    a, b = np.empty((m, k), CI8), np.empty((k, n), CI8)
    for x in (a, b):
        x['re'] = -128
        x['im'] = -128
    la = LinAlg()
    for ca in (False, True):
        for cb in (False, True):
            gold = ab_gold(a, b, ca, cb)
            assert np.abs(gold).max() == np.float32(2 * k * 2 ** 14)
            np.testing.assert_array_equal(ab_dev(la, a, b, ca, cb), gold, err_msg=str((ca, cb)))


def test_ab_staging_buffer_regrow():
    """One handle across a large, a small and a larger call: the a^T staging
    buffer is reused, then regrown."""
    rng = np.random.default_rng(23)
    la = LinAlg()
    for m, n, k in [(200, 256, 600), (5, 8, 10), (300, 128, 900)]:
        a, b = full_range_ci8(rng, (m, k)), full_range_ci8(rng, (k, n))
        da, db = bf.asarray(a, space='cuda'), bf.asarray(b, space='cuda')
        dc = bf.zeros((m, n), 'cf32', 'cuda')
        before = bf.launch_count()
        la.matmul(1, da, db, 0, dc)
        assert bf.launch_count() - before == 2, "the tensor-core path was not taken"
        np.testing.assert_array_equal(np.asarray(dc.copy('system')), ab_gold(a, b), err_msg=str((m, n, k)))


# ------------------------------------------------------------ status codes
def test_correlator_status_codes():
    h = LinAlg()

    def status(x, c):
        return _bf.bfLinAlgMatMul(h.obj, 1.0, None, x.as_BFarray(), 0.0, c.as_BFarray())

    assert status(bf.zeros((8, 16), 'ci4', 'cuda'), bf.zeros((16, 16), 'cf32', 'cuda')) == \
        _bf.BF_STATUS_UNSUPPORTED_DTYPE
    d_big = bf.zeros((16, 32), 'cf32', 'cuda')
    assert status(bf.zeros((8, 16), 'ci8', 'cuda'), d_big[:, ::2]) == _bf.BF_STATUS_UNSUPPORTED_STRIDE
    assert status(bf.zeros((65536, 1, 1), 'ci8', 'cuda'), bf.zeros((65536, 1, 1), 'cf32', 'cuda')) == \
        _bf.BF_STATUS_UNSUPPORTED_SHAPE
