"""bfLinAlgMatMul (correlator forms) parity.  CPU: the oracle against the
closed-form case of the reference's pipeline test (test/test_pipeline.py:66-72,
258-298).  GPU: tensor-core path and SIMT fallback against the oracle --
integer-exact -- over the sweep of test/test_linalg.py:221-240 (odd sizes,
misaligned views) and BASELINE config 4 shapes; upper triangle untouched;
beta accumulation; a.a^H form."""
import os

import numpy as np
import pytest

import bifrost_b200 as bf
from bifrost_b200.linalg import LinAlg
from oracle import linalg as olinalg

CI8 = bf.DataType('ci8').as_numpy_dtype()


def closed_form_input(ntime, nchan, nstand, npol):
    """CorrelateTestInputBlock of the reference (test/test_pipeline.py:66-72)."""
    i = np.arange(nstand * npol * 2) % 255 - 127
    x = np.empty((ntime, nchan, nstand * npol), dtype=CI8)
    x['re'] = i[0::2]
    x['im'] = i[1::2]
    return x


def test_oracle_reproduces_reference_closed_form():
    ntime, nchan, nstand, npol = 12, 3, 10, 2
    x = closed_form_input(ntime, nchan, nstand, npol)
    got = olinalg.correlate(np.transpose(x, (1, 0, 2)))
    i = np.arange(nstand * npol * 2) % 255 - 127
    v = (i[0::2] + 1j * i[1::2]).astype(np.complex64)
    expected = ntime * v[:, None].conj() * v[None, :]
    triu = np.triu_indices(nstand * npol, 1)
    expected[triu] = 0
    np.testing.assert_allclose(got, np.broadcast_to(expected, got.shape), rtol=1e-6)


def rand_ci8(rng, shape):
    x = np.empty(shape, dtype=CI8)
    x['re'] = rng.integers(-127, 128, size=shape)
    x['im'] = rng.integers(-127, 128, size=shape)
    return x


def run_bhb(x_tcn, beta=0.0, alpha=1.0, c0=None, perm=(1, 0, 2)):
    """x_tcn: [ntime, nchan, n] host array; correlate over time per channel."""
    d_x = bf.asarray(x_tcn, space='cuda')
    xv = d_x.transpose(perm)
    nchan, n = x_tcn.shape[1], x_tcn.shape[2]
    c_init = np.zeros((nchan, n, n), np.complex64) if c0 is None else c0
    d_c = bf.asarray(c_init, space='cuda')
    LinAlg().matmul(alpha, None, xv, beta, d_c)
    return np.asarray(d_c.copy('system'))


@pytest.mark.gpu
@pytest.mark.parametrize("ntime,nchan,n", [(512, 4, 512), (100, 3, 128), (64, 2, 64), (1000, 1, 72),
                                           (8, 5, 200), (33, 2, 16), (129, 1, 136), (65, 1, 704),
                                           (193, 2, 1024)])
def test_tensor_core_path_is_integer_exact(ntime, nchan, n):
    rng = np.random.default_rng(ntime + n)
    x = rand_ci8(rng, (ntime, nchan, n))
    sentinel = (np.arange(nchan * n * n).reshape(nchan, n, n) % 7 + 1j).astype(np.complex64)
    got = run_bhb(x, c0=sentinel)
    want = olinalg.correlate(np.transpose(x, (1, 0, 2)), c=sentinel)
    np.testing.assert_array_equal(got, want)          # incl. untouched upper triangle


@pytest.mark.gpu
def test_tensor_core_equals_simt_fallback():
    rng = np.random.default_rng(5)
    x = rand_ci8(rng, (300, 3, 256))
    a = run_bhb(x)
    os.environ['BFB_LINALG_SIMT'] = '1'
    try:
        b = run_bhb(x)
    finally:
        del os.environ['BFB_LINALG_SIMT']
    np.testing.assert_array_equal(a, b)


@pytest.mark.gpu
def test_reference_sweep_small_and_misaligned():
    """test/test_linalg.py:221-240 (subset): nstand 1..65 x ntime x nchan x misalign."""
    rng = np.random.default_rng(1234)
    for nstand in [1, 2, 3, 4, 5, 8, 9, 16, 17, 31, 32, 33, 64, 65]:
        for ntime in [1, 2, 3, 4, 8, 12]:
            for nchan in [1, 2, 5]:
                for mis in [0, 2]:
                    n_full = nstand * 2
                    x = rand_ci8(rng, (ntime, nchan, n_full))
                    d_x = bf.asarray(x, space='cuda')
                    xv = d_x.transpose(1, 0, 2)[..., mis:]
                    n = n_full - mis
                    if n <= 0:
                        continue
                    d_c = bf.zeros((nchan, n, n), 'cf32', 'cuda')
                    LinAlg().matmul(1, None, xv, 0, d_c)
                    got = np.asarray(d_c.copy('system'))
                    want = olinalg.correlate(np.transpose(x, (1, 0, 2))[..., mis:])
                    np.testing.assert_array_equal(got, want, err_msg=str((nstand, ntime, nchan, mis)))


@pytest.mark.gpu
def test_beta_alpha_and_batch_dims():
    rng = np.random.default_rng(6)
    x1, x2 = rand_ci8(rng, (128, 2, 64)), rand_ci8(rng, (128, 2, 64))
    c = run_bhb(x1)
    c = run_bhb(x2, beta=1.0, c0=c)
    want = olinalg.correlate(np.transpose(x2, (1, 0, 2)), c=olinalg.correlate(np.transpose(x1, (1, 0, 2))), beta=1.0)
    np.testing.assert_array_equal(c, want)
    c2 = run_bhb(x1, alpha=0.5)
    np.testing.assert_array_equal(c2, olinalg.correlate(np.transpose(x1, (1, 0, 2)), alpha=0.5))
    # extra leading batch dim: [beam, chan, time, n]
    xb = rand_ci8(rng, (3, 64, 4, 48))                # [beam, time, chan, n]
    d_x = bf.asarray(xb, space='cuda')
    xv = d_x.transpose(0, 2, 1, 3)
    d_c = bf.zeros((3, 4, 48, 48), 'cf32', 'cuda')
    LinAlg().matmul(1, None, xv, 0, d_c)
    np.testing.assert_array_equal(np.asarray(d_c.copy('system')),
                                  olinalg.correlate(np.transpose(xb, (0, 2, 1, 3))))


@pytest.mark.gpu
def test_aah_form_and_float_inputs():
    rng = np.random.default_rng(7)
    a = rand_ci8(rng, (2, 24, 100))                   # [batch, n, ntime]
    d_a = bf.asarray(a, space='cuda')
    d_c = bf.zeros((2, 24, 24), 'cf32', 'cuda')
    LinAlg().matmul(1, d_a, None, 0, d_c)
    av = a['re'].astype(np.float64) + 1j * a['im']
    full = av @ np.swapaxes(av.conj(), -1, -2)
    il = np.tril_indices(24)
    want = np.zeros((2, 24, 24), np.complex64)
    want[..., il[0], il[1]] = full[..., il[0], il[1]]
    np.testing.assert_array_equal(np.asarray(d_c.copy('system')), want)
    xf = (rng.normal(size=(3, 200, 40)) + 1j * rng.normal(size=(3, 200, 40))).astype(np.complex64)
    d_cf = bf.zeros((3, 40, 40), 'cf32', 'cuda')
    LinAlg().matmul(1, None, bf.asarray(xf, space='cuda'), 0, d_cf)
    np.testing.assert_allclose(np.asarray(d_cf.copy('system')), olinalg.correlate(xf), rtol=1e-4, atol=1e-3)


@pytest.mark.gpu
def test_correlate_block_closed_form():
    """The reference's pipeline test for CorrelateBlock (test/test_pipeline.py:230-298)."""
    from bifrost_b200 import blocks
    from bifrost_b200.pipeline import Pipeline
    ntime, nchan, nstand, npol = 96, 4, 16, 2
    x = closed_form_input(ntime, nchan, nstand, npol).reshape(ntime, nchan, nstand, npol)
    hdr = {'_tensor': {'dtype': 'ci8', 'shape': [-1, nchan, nstand, npol],
                       'labels': ['time', 'freq', 'station', 'pol'],
                       'scales': [[0, 1e-3], [100.0, 0.1], None, None], 'units': ['s', 'MHz', None, None]},
           'name': 'corr', 'gulp_nframe': 32}
    chunks = []
    with Pipeline() as p:
        src = blocks.array_source(x, hdr, gulp_nframe=32)
        b = blocks.copy(src, space='cuda')
        b = blocks.correlate(b, nframe_per_integration=96)
        b = blocks.copy(b, space='system')
        blocks.callback_sink(b, None, lambda s: chunks.append(np.array(s.data)))
        p.run()
    got = chunks[0].reshape(nchan, nstand * npol, nstand * npol)
    i = np.arange(nstand * npol * 2) % 255 - 127
    v = (i[0::2] + 1j * i[1::2]).astype(np.complex64)
    expected = ntime * v[:, None].conj() * v[None, :]
    il = np.tril_indices(nstand * npol)
    np.testing.assert_allclose(got[:, il[0], il[1]], np.broadcast_to(expected[il], (nchan, len(il[0]))), rtol=1e-6)


def H(x):
    """Conjugate transpose of the last two axes as a view (test/test_linalg.py:41-43)."""
    axes = list(range(x.ndim))
    axes[-1], axes[-2] = axes[-2], axes[-1]
    return x.transpose(axes).conj()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.complex64, np.complex128])
@pytest.mark.parametrize("transpose", [False, True])
def test_matmul_ab_float_types(dtype, transpose):
    """test/test_linalg.py:110-135,275-285: c = a.b for real / complex floats, incl. H views."""
    rng = np.random.default_rng(7)
    for shape, k in [((11, 23), 7), ((11, 23), 23), ((5, 11, 23), 11), ((3, 64, 40), 33)]:
        ashape, bshape = shape[:-2] + (shape[-2], k), shape[:-2] + (k, shape[-1])
        a = (rng.random(ashape) * 127).astype(dtype)
        b = (rng.random(bshape) * 127).astype(dtype)
        if np.iscomplexobj(a):
            a = a + 1j * (rng.random(ashape) * 50).astype(dtype)
            b = b - 1j * (rng.random(bshape) * 50).astype(dtype)
        ga, gb = (np.conj(np.swapaxes(b, -1, -2)), np.conj(np.swapaxes(a, -1, -2))) if transpose else (a, b)
        want = np.matmul(ga, gb)
        da, db = bf.asarray(a, space='cuda'), bf.asarray(b, space='cuda')
        if transpose:
            da, db = H(db), H(da)
        dc = bf.asarray(np.zeros_like(want), space='cuda')
        LinAlg().matmul(1, da, db, 0, dc)
        np.testing.assert_allclose(np.asarray(dc.copy('system')), want, rtol=1e-4, atol=1e-5 * np.abs(want).max())


@pytest.mark.gpu
def test_matmul_ab_ci8_and_beamformer():
    """test/test_linalg.py:90-109 (ci8 x ci8) and :136-150 (cf32 weights x ci8 voltages)."""
    rng = np.random.default_rng(8)
    m, n, k = 111, 223, 77
    a = rand_ci8(rng, (m, k))
    b = rand_ci8(rng, (k, n))
    af = a['re'].astype(np.float32) + 1j * a['im'].astype(np.float32)
    bfl = b['re'].astype(np.float32) + 1j * b['im'].astype(np.float32)
    dc = bf.zeros((m, n), 'cf32', 'cuda')
    LinAlg().matmul(1, bf.asarray(a, space='cuda'), bf.asarray(b, space='cuda'), 0, dc)
    np.testing.assert_array_equal(np.asarray(dc.copy('system')), (af @ bfl).astype(np.complex64))
    ntime, nbeam, nstand, nchan = 64, 5, 32, 3
    x = rand_ci8(rng, (ntime, nchan, nstand * 2))
    xf = x['re'].astype(np.float32) + 1j * x['im'].astype(np.float32)
    w = (rng.integers(-127, 128, size=(nbeam, nchan, nstand * 2)) +
         1j * rng.integers(-127, 128, size=(nbeam, nchan, nstand * 2))).astype(np.complex64)
    want = np.matmul(w.transpose(1, 0, 2), xf.transpose(1, 2, 0))
    d_x, d_w = bf.asarray(x, space='cuda'), bf.asarray(w, space='cuda')
    d_b = bf.zeros(want.shape, 'cf32', 'cuda')
    LinAlg().matmul(1, d_w.transpose((1, 0, 2)), d_x.transpose((1, 2, 0)), 0, d_b)
    np.testing.assert_allclose(np.asarray(d_b.copy('system')), want, rtol=1e-5)
    # beta path
    LinAlg().matmul(0.5, d_w.transpose((1, 0, 2)), d_x.transpose((1, 2, 0)), 2.0, d_b)
    np.testing.assert_allclose(np.asarray(d_b.copy('system')), 2.5 * want, rtol=1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,k,batch", [(5, 64, 32, None), (64, 128, 64, None), (111, 224, 77, None),
                                         (65, 136, 500, 3), (200, 1000, 300, 2), (32, 4096, 512, 4)])
def test_matmul_ab_ci8_on_the_tensor_cores(m, n, k, batch):
    """ci8 x ci8 -> cf32 with TMA-friendly operands takes the wgmma kernel
    (two launches: a^T staging + the product); exact integers, every
    conjugation flag, alpha / beta, a shared or per-batch weight matrix."""
    rng = np.random.default_rng(m * n + k)
    bs = () if batch is None else (batch,)
    a = rand_ci8(rng, bs + (m, k))
    b = rand_ci8(rng, bs + (k, n))
    ar, ai = a['re'].astype(np.int64), a['im'].astype(np.int64)
    br, bi = b['re'].astype(np.int64), b['im'].astype(np.int64)

    def gold(ca, cb):
        sa, sb = (-1 if ca else 1), (-1 if cb else 1)
        re = ar @ br - (sa * ai) @ (sb * bi)
        im = ar @ (sb * bi) + (sa * ai) @ br
        return (re + 1j * im).astype(np.complex64)

    da, db = bf.asarray(a, space='cuda'), bf.asarray(b, space='cuda')
    la = LinAlg()
    for ca in (False, True):
        for cb in (False, True):
            dc = bf.asarray(np.full(bs + (m, n), 7 - 3j, np.complex64), space='cuda')
            before = bf.launch_count()
            la.matmul(1, da.conj() if ca else da, db.conj() if cb else db, 0, dc)
            assert bf.launch_count() - before == 2, "the tensor-core path was not taken"
            np.testing.assert_array_equal(np.asarray(dc.copy('system')), gold(ca, cb))
    # alpha / beta
    c0 = (rng.integers(-50, 50, size=bs + (m, n)) + 1j * rng.integers(-50, 50, size=bs + (m, n))).astype(np.complex64)
    dc = bf.asarray(c0, space='cuda')
    la.matmul(0.5, da, db, 2.0, dc)
    np.testing.assert_allclose(np.asarray(dc.copy('system')), 0.5 * gold(False, False) + 2.0 * c0, rtol=1e-6)
    # one weight matrix for every batch entry (broadcast batch dim of a)
    if batch is not None:
        a1 = bf.asarray(a[:1], space='cuda')
        dc = bf.zeros(bs + (m, n), 'cf32', 'cuda')
        la.matmul(1, a1, db, 0, dc)
        ar, ai = np.broadcast_to(ar[:1], ar.shape), np.broadcast_to(ai[:1], ai.shape)
        np.testing.assert_array_equal(np.asarray(dc.copy('system')), gold(False, False))
    # same numbers from the SIMT kernel
    os.environ['BFB_LINALG_SIMT'] = '1'
    try:
        dc2 = bf.zeros(bs + (m, n), 'cf32', 'cuda')
        la.matmul(1, da if batch is None else bf.asarray(a[:1], space='cuda'), db, 0, dc2)
    finally:
        del os.environ['BFB_LINALG_SIMT']
    np.testing.assert_array_equal(np.asarray(dc2.copy('system')), gold(False, False))


@pytest.mark.gpu
def test_invalid_forms_return_status():
    from bifrost_b200.libbifrost import _bf
    a = bf.empty((4, 8), 'cf32', 'cuda')
    b = bf.empty((9, 4), 'cf32', 'cuda')
    c = bf.empty((4, 4), 'cf32', 'cuda')
    h = LinAlg()
    assert _bf.bfLinAlgMatMul(h.obj, 1.0, a.as_BFarray(), b.as_BFarray(), 0.0, c.as_BFarray()) == \
        _bf.BF_STATUS_INVALID_SHAPE
    assert _bf.bfLinAlgMatMul(h.obj, 1.0, None, None, 0.0, c.as_BFarray()) == _bf.BF_STATUS_INVALID_ARGUMENT


@pytest.mark.gpu
@pytest.mark.parametrize("ntime", [512, 2048, 8192])
def test_baseline_config4_full_size_against_the_oracle(ntime):
    """BASELINE config 4 at its real size: x ci8 [ntime, 512 chan, 256 stand x 2 pol],
    C cf32 [512, 512, 512] (the shape bench / tools/bench_ops.py time), value-checked
    on a channel subset -- integer-exact -- against oracle/linalg.py.  |C| stays
    below 2^24 only for ntime <= 512 with full-range int8, so the longer
    integrations draw from [-31, 31] (sums < 2^24: fp32-exact on both sides)."""
    import torch
    nchan, n = 512, 512
    amp = 127 if ntime <= 512 else 31
    g = torch.Generator(device='cuda').manual_seed(ntime)
    raw = torch.randint(-amp, amp + 1, (ntime, nchan, n, 2), dtype=torch.int8, device='cuda', generator=g)
    d_x = bf.ndarray(space='cuda', shape=(ntime, nchan, n), dtype='ci8', buffer=raw.data_ptr())   # zero-copy view
    d_c = bf.zeros((nchan, n, n), 'cf32', 'cuda')
    LinAlg().matmul(1, None, d_x.transpose((1, 0, 2)), 0, d_c)
    chans = [0, 1, 255, 256, 300, 511]
    got = np.stack([np.asarray(d_c[c:c + 1].copy('system'))[0] for c in chans])
    sub = raw[:, chans].cpu().numpy()                                      # [ntime, 6, n, 2]
    x = np.empty((len(chans), ntime, n), dtype=CI8)
    x['re'] = np.transpose(sub[..., 0], (1, 0, 2))
    x['im'] = np.transpose(sub[..., 1], (1, 0, 2))
    want = olinalg.correlate(x)
    np.testing.assert_array_equal(got, want)


@pytest.mark.gpu
def test_correlator_matches_the_reference_library():
    """The same inputs through the reference's own bfLinAlgMatMul
    (src/linalg.cu:242-357 + linalg_kernels.cu) gave the stored outputs
    (tests/golden/make_ref_gpu_golden.py); ours against them."""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from golden import make_ref_gpu_golden as refgold
    gold = refgold.load()
    for ci, x in enumerate(refgold.linalg_inputs()):
        ntime = x.shape[0]
        ours = refgold.linalg_lower(run_bhb(x)).ravel()
        a = ours[refgold.sample_index(ours.size, 2000 + ci)]
        b = gold['linalg/%d' % ci]
        # The reference accumulates (x/127)(y/127) in fp32 and rounds x127^2 at the end
        # (linalg_kernels.cu:94-112): exact only while the rounding errors stay below
        # one half -- short integrations.  Ours is integer-exact (checked against the
        # oracle above); the long case agrees to the reference's own fp32 accuracy.
        if ntime <= 64:
            np.testing.assert_array_equal(a, b)
        else:
            np.testing.assert_allclose(a, b, rtol=2e-5, atol=2.0)
