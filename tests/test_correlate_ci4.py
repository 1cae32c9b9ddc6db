"""The correlator on ci4 input (one byte per complex sample, high nibble real,
both nibbles two's complement): bfLinAlgCorrelateCi4 (the a.a^H / b^H.b forms
of bfLinAlgMatMul for ci4), bfLinAlgCorrelateCi4ToStorage, LinAlg (which
routes ci4 there) and blocks.correlate.  bfLinAlgMatMul and
bfLinAlgCorrelateToStorage keep the reference's status for ci4.

A ci4 correlation is defined as the ci8 correlation of the same complex
integers, bit for bit.  Every GPU case compares with the ci8 call on the
decoded values (and with oracle/linalg.py on them), and asserts which kernel
ran: corr4_tc_kernel / corr4_storage_tc_kernel on the tensor cores, the SIMT
kernel for layouts TMA cannot describe.  The ci4 sums are exact in int32 up
to 2^24 - 1 samples, so one pass covers integrations the ci8 kernels split.

CPU: the ci4 reference against numpy, the block's header, and a no-spill
sm_90a build of the new kernels."""
import contextlib
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
from oracle import beamform as obeamform
from oracle import linalg as olinalg
from oracle import visibilities as ovis

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CI4 = bf.DataType('ci4').as_numpy_dtype()
CI8 = bf.DataType('ci8').as_numpy_dtype()
TC4 = 'corr4_tc_kernel'
FUSED4 = 'corr4_storage_tc_kernel'


# ------------------------------------------------------------------ helpers
def make_ci4(re_, im_):
    """Structured ci4 from explicit nibble values in [-8, 7] (bf.DataType's
    convention: high nibble real)."""
    x = np.empty(np.shape(re_), CI4)
    x['re_im'] = ((np.asarray(re_) & 0xF) << 4 | (np.asarray(im_) & 0xF)).astype(np.uint8)
    return x


def full_range_ci4(rng, shape):
    """Uniform over [-8, 7], with -8 forced into whole rows: every station of
    some time samples (real part) and every sample of station 0 (both parts)."""
    re_ = rng.integers(-8, 8, size=shape)
    im_ = rng.integers(-8, 8, size=shape)
    re_[3::5] = -8
    re_[..., 0] = -8
    im_[..., 0] = -8
    return make_ci4(re_, im_)


def decoded_ci8(x4):
    """The same complex integers as ci8, decoded by the oracle's ci4 decoder."""
    re_, im_, _ = obeamform._components(x4, False)
    x8 = np.empty(x4.shape, CI8)
    x8['re'], x8['im'] = re_, im_
    return x8


def oracle_ci4(u4, c=None, alpha=1.0, beta=0.0):
    """oracle/linalg.correlate of u4's decoded values (u4: [..., ntime, n] ci4)."""
    return olinalg.correlate(decoded_ci8(u4), c=c, alpha=alpha, beta=beta)


def sentinel(shape):
    return (np.arange(int(np.prod(shape))).reshape(shape) % 7 + 0.5 - 3j).astype(np.complex64)


def bits(a):
    return np.ascontiguousarray(a, np.complex64).view(np.uint64)


def same_bits(got, want, msg=''):
    got, want = bits(got), bits(want)
    assert got.shape == want.shape, msg
    bad = got != want
    assert not bad.any(), "%s: %i of %i differ, first at %s" % (msg, bad.sum(), bad.size, np.argwhere(bad)[0])


def host(d):
    return np.asarray(d.copy('system'))


def short(name):
    """'void bfb::corr4_tc_kernel(...)' -> 'corr4_tc_kernel'."""
    m = re.search(r'(\w+)(<[^()]*>)?\(', name)
    return m.group(1) if m else name


@contextlib.contextmanager
def forced_simt(on=True):
    if on:
        os.environ['BFB_LINALG_SIMT'] = '1'
    try:
        yield
    finally:
        if on:
            del os.environ['BFB_LINALG_SIMT']


def ran(fn, reset=None):
    from kernel_trace import device_kernels
    return [short(k) for k in device_kernels(fn, reset=reset)]


def corr_paths(names):
    """'tc' / 'simt' for each correlator kernel among `names`."""
    return ['tc' if k == TC4 else 'simt' for k in names if k in (TC4, 'corr_simt_kernel')]


def correlate_dev(xv, c, alpha=1.0, beta=0.0, aah=False, simt=False):
    """c <- alpha xv^H.xv (or xv.xv^H) + beta c on the device: c on the host
    and the kernels that ran."""
    la = LinAlg()
    c0 = host(c)

    def reset():
        c[...] = c0
    with forced_simt(simt):
        names = ran(lambda: la.matmul(alpha, xv if aah else None, None if aah else xv, beta, c), reset=reset)
    return host(c), names


# ---------------------------------------------------------------------- CPU
def test_reference_equals_numpy_and_ci8_over_the_full_nibble_range():
    """Every byte value appears; -8 fills whole rows (time samples) and whole
    columns (stations) in both parts.  The ci4 reference is numpy's complex128
    x^H x rounded once to complex64, and the ci8 reference of the decoded values."""
    rng = np.random.default_rng(1)
    nchan, ntime, n = 2, 300, 40
    raw = rng.integers(0, 256, size=(nchan, ntime, n)).astype(np.uint8)
    raw[:, :256, 5] = np.arange(256)
    raw[:, 7] = 0x88
    raw[:, :, 9] = 0x88
    x4 = raw.view(CI4)
    re_ = (raw.astype(np.int8) >> 4).astype(np.int64)
    im_ = ((raw << 4).astype(np.int8) >> 4).astype(np.int64)
    assert re_.min() == im_.min() == -8 and re_.max() == im_.max() == 7
    assert (re_[:, 7] == -8).all() and (im_[:, :, 9] == -8).all()
    xc = re_ + 1j * im_
    want = (np.swapaxes(xc.conj(), -1, -2) @ xc).astype(np.complex64)
    got = oracle_ci4(x4)
    il = np.tril_indices(n)
    same_bits(got[:, il[0], il[1]], want[:, il[0], il[1]])
    iu = np.triu_indices(n, 1)
    assert (got[:, iu[0], iu[1]] == 0).all()                 # the upper triangle is kept
    same_bits(got, olinalg.correlate(decoded_ci8(x4)))
    assert np.array_equal(make_ci4(re_, im_)['re_im'], raw)


def test_block_header_is_the_ci8_header():
    from bifrost_b200.blocks.correlate import CorrelateBlock

    class Seq(object):
        def __init__(self, header):
            self.header = header
    heads = []
    for dtype in ('ci4', 'ci8'):
        hdr = volt_header(3, 5, dtype, gulp=4)
        for output in ('matrix', 'storage'):
            with Pipeline():
                src = blocks.array_source(np.zeros((4, 3, 5, 2), CI8), volt_header(3, 5, 'ci8', 4), gulp_nframe=4)
                b = CorrelateBlock(src, 8, output=output)
            heads.append(b.on_sequence(Seq(hdr)))
    assert heads[:2] == heads[2:]


def test_ci4_kernels_compile_without_spills(tmp_path):
    """corr4_tc_kernel, corr4_storage_tc_kernel and the ci4 SIMT kernel: one
    entry each, sm_90a, no spills."""
    src = os.path.join(ROOT, 'bifrost_b200', 'csrc')
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    out = subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17',
                          '-I' + os.path.join(ROOT, 'include'), '-I' + src, '--expt-relaxed-constexpr',
                          '-Xptxas', '-v', '-c', os.path.join(src, 'linalg.cu'), '-o', str(tmp_path / 'l.o')],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    stats, entry = {}, None
    for line in out.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            entry = m.group(1)
        elif entry and 'spill stores' in line:
            stats[entry] = line
    for name in ('15corr4_tc_kernel', '23corr4_storage_tc_kernel', 'corr_simt_kernelINS_3Ci4EiEE'):
        got = {k: v for k, v in stats.items() if name in k}
        assert len(got) == 1, (name, list(stats))
        assert all(' 0 bytes spill stores, 0 bytes spill loads' in v for v in got.values()), got


# ------------------------------------------------------- GPU: shape sweep
# The ci8 sweep's n (row-block counts 1..8, 11 and 16, odd and even, below
# one box) and ntime (slab tails, stage-ring wraps), nchan 1 and 3, in the
# ring-frame layout [time][chan][n] viewed as [chan][time][n].
SWEEP_N = [16, 24, 56, 64, 72, 120, 128, 136, 192, 200, 256, 264, 320, 384, 392, 448, 512, 704, 1024]
SWEEP_NTIME = [1, 8, 63, 64, 65, 191, 192, 193, 640]
# n that do not reach the tensor cores: n bytes per station row is not a
# multiple of 16, so neither is the time stride (nor, for nchan 3, the
# channel stride) and TMA cannot describe the layout.
SWEEP_SIMT = {n for n in SWEEP_N if n % 16}


@pytest.mark.gpu
@pytest.mark.parametrize("n", SWEEP_N)
def test_sweep_equals_ci8_and_oracle(n):
    rng = np.random.default_rng(4000 + n)
    cases = [(ntime, nchan) for ntime in SWEEP_NTIME for nchan in (1, 3)]
    xs = [full_range_ci4(rng, (ntime, nchan, n)) for ntime, nchan in cases]
    d_x4 = [bf.asarray(bf.ndarray(x, dtype='ci4'), space='cuda') for x in xs]
    d_x8 = [bf.asarray(decoded_ci8(x), space='cuda') for x in xs]
    la = LinAlg()
    got = {}
    for simt in (False, True):
        d_cs = [bf.asarray(sentinel((nchan, n, n)), space='cuda') for _, nchan in cases]

        def run():
            for d_x, d_c in zip(d_x4, d_cs):
                la.matmul(1, None, d_x.transpose((1, 0, 2)), 0, d_c)
        with forced_simt(simt):
            paths = corr_paths(ran(run))
        want_paths = ['simt' if simt or n in SWEEP_SIMT else 'tc' for _ in cases]
        assert paths == want_paths, list(zip(cases, paths))
        got[simt] = [host(d_c) for d_c in d_cs]
    d_cs = [bf.asarray(sentinel((nchan, n, n)), space='cuda') for _, nchan in cases]
    for d_x, d_c in zip(d_x8, d_cs):
        la.matmul(1, None, d_x.transpose((1, 0, 2)), 0, d_c)
    for (ntime, nchan), x, tc, simt, c8 in zip(cases, xs, got[False], got[True], d_cs):
        msg = str((n, ntime, nchan))
        same_bits(tc, oracle_ci4(np.transpose(x, (1, 0, 2)), c=sentinel((nchan, n, n))), msg)
        same_bits(tc, host(c8), msg)
        same_bits(simt, tc, msg)


# ------------------------------------------ GPU: forms, views, alpha / beta
@pytest.mark.gpu
@pytest.mark.parametrize("case", ['aah', 'conj', 'alpha_beta', 'aah_conj'])
def test_forms_and_arguments_equal_ci8(case):
    """Each call, on ci4 and on the decoded ci8 with the same arguments, onto
    the same sentinel c: identical bits, the upper triangle untouched."""
    rng = np.random.default_rng(7)
    nchan, ntime, n = 3, 193, 128
    aah = case.startswith('aah')
    shape = (nchan, n, ntime) if aah else (ntime, nchan, n)
    x4 = full_range_ci4(rng, shape)
    alpha, beta = (0.5, 2.0) if case in ('alpha_beta', 'aah') else (1.0, 0.0)
    outs = []
    for x in (bf.ndarray(x4, dtype='ci4'), decoded_ci8(x4)):
        d_x = bf.asarray(x, space='cuda')
        xv = d_x if aah else d_x.transpose((1, 0, 2))
        if 'conj' in case:
            xv = xv.conj()
        got, names = correlate_dev(xv, bf.asarray(sentinel((nchan, n, n)), space='cuda'), alpha, beta, aah=aah)
        outs.append((got, names))
    (g4, k4), (g8, _) = outs
    assert corr_paths(k4) == ['simt' if aah else 'tc'], k4
    same_bits(g4, g8)
    iu = np.triu_indices(n, 1)
    same_bits(g4[:, iu[0], iu[1]], sentinel((nchan, n, n))[:, iu[0], iu[1]])


@pytest.mark.gpu
def test_misaligned_base_falls_back_to_simt_with_the_same_bits():
    """[time][chan][n] ring frames inside a padded buffer; the view starts one
    element (1 B) in, so TMA cannot take it."""
    rng = np.random.default_rng(8)
    nchan, ntime, n = 3, 130, 64
    pad = full_range_ci4(rng, (ntime, nchan, n + 16))
    d_pad = bf.asarray(bf.ndarray(pad, dtype='ci4'), space='cuda')
    d_al = bf.asarray(bf.ndarray(np.ascontiguousarray(pad[:, :, 1:n + 1]), dtype='ci4'), space='cuda')
    got_mis, names_mis = correlate_dev(d_pad[:, :, 1:n + 1].transpose((1, 0, 2)),
                                       bf.zeros((nchan, n, n), 'cf32', 'cuda'))
    got_al, names_al = correlate_dev(d_al.transpose((1, 0, 2)), bf.zeros((nchan, n, n), 'cf32', 'cuda'))
    assert corr_paths(names_mis) == ['simt'] and corr_paths(names_al) == ['tc']
    same_bits(got_mis, got_al)
    same_bits(got_al, oracle_ci4(np.transpose(pad[:, :, 1:n + 1], (1, 0, 2))))


@pytest.mark.gpu
def test_agrees_with_bfunpack_to_ci8():
    """bfUnpack reads the byte-reversed nibble order; unpacking the
    byte-reversed array gives the ci8 whose correlation the ci4 one equals."""
    rng = np.random.default_rng(9)
    nchan, ntime, n = 2, 100, 48
    x4 = full_range_ci4(rng, (ntime, nchan, n))
    d4 = bf.asarray(bf.ndarray(x4, dtype='ci4'), space='cuda')
    d8 = bf.empty((ntime, nchan, n), 'ci8', 'cuda')
    bf.unpack(bf.asarray(bf.ndarray(x4, dtype='ci4').byteswap(), space='cuda'), d8)
    x8 = host(d8)
    assert np.array_equal(x8['re'], decoded_ci8(x4)['re']) and np.array_equal(x8['im'], decoded_ci8(x4)['im'])
    g4, k4 = correlate_dev(d4.transpose((1, 0, 2)), bf.zeros((nchan, n, n), 'cf32', 'cuda'))
    g8, _ = correlate_dev(d8.transpose((1, 0, 2)), bf.zeros((nchan, n, n), 'cf32', 'cuda'))
    assert corr_paths(k4) == ['tc']
    same_bits(g4, g8)


# --------------------------------------------------- GPU: long integrations
@pytest.mark.gpu
def test_past_the_ci8_one_pass_limit_is_one_launch():
    """200000 samples: the ci8 kernel would need two passes, ci4 takes one."""
    rng = np.random.default_rng(10)
    ntime, n = 200000, 32
    x4 = full_range_ci4(rng, (ntime, 1, n))
    got, names = correlate_dev(bf.asarray(bf.ndarray(x4, dtype='ci4'), space='cuda').transpose((1, 0, 2)),
                               bf.zeros((1, n, n), 'cf32', 'cuda'))
    assert corr_paths(names) == ['tc']
    same_bits(got, oracle_ci4(np.transpose(x4, (1, 0, 2))))


@pytest.mark.gpu
def test_one_past_the_ci4_bound_all_minus_8():
    """2^24 samples of -8-8i at n = 64 (1.07 GB): 2^24 - 1 samples in one
    pass, then one more with beta = 1.  conj(-8-8i)(-8-8i) = 128, so every
    lower-triangle entry is 128 * 2^24 = 2^31 + 0i; the first chunk's
    128 (2^24 - 1) and the sum are both exact in fp32, so an int32 overflow or
    a second rounding would show."""
    import time
    import torch
    ntime, n = 2 ** 24, 64
    buf = torch.full((ntime * n,), 0x88, dtype=torch.uint8, device='cuda')
    xv = bf.ndarray(space='cuda', shape=(1, ntime, n), dtype='ci4', buffer=buf.data_ptr(), strides=(ntime * n, n, 1))
    d_c = bf.zeros((1, n, n), 'cf32', 'cuda')
    t0 = time.perf_counter()
    got, names = correlate_dev(xv, d_c)
    print("ci4 correlation of %d samples at n = %d: %.3f s including the kernel trace" %
          (ntime, n, time.perf_counter() - t0))
    assert names == [TC4, TC4], names
    il = np.tril_indices(n)
    low = got[0][il]
    assert (low.real == np.float32(2 ** 31)).all() and (low.imag == 0).all()
    iu = np.triu_indices(n, 1)
    assert (got[0][iu] == 0).all()
    del buf


# --------------------------------------------- GPU: correlate to storage
def storage_two_calls(la, xv, nchan, nstand):
    n = 2 * nstand
    d_c = bf.empty((nchan, n, n), 'cf32', 'cuda')
    d_s = bf.empty((nstand * (nstand + 1) // 2, nchan, 4), 'cf32', 'cuda')
    la.matmul(1, None, xv, 0, d_c)
    bf.visibilities.to_storage(d_c.reshape(nchan, nstand, 2, nstand, 2), d_s)
    return host(d_s)


def storage_call(la, xv, nchan, nstand, padded):
    nb = nstand * (nstand + 1) // 2
    fill = np.complex64(1234.5 - 678.25j)
    if padded:
        d_base = bf.asarray(np.full((nb + 1, nchan + 2, 4), fill, np.complex64), space='cuda')
        view = np.s_[1:, 1:nchan + 1]
    else:
        d_base = bf.asarray(np.full((nb, nchan, 4), np.nan, np.complex64), space='cuda')
        view = np.s_[...]
    names = ran(lambda: la.correlate_to_storage(xv, d_base[view]))
    got = host(d_base)
    if padded:
        pad = np.ones(got.shape, bool)
        pad[view] = False
        assert (got[pad] == fill).all()
    return got[view], names


# (nstand, nchan, ntime, padded vis, conjugated view)
STORAGE_CASES = [(8, 3, 1, False, False), (16, 3, 65, True, False), (32, 1, 640, False, False),
                 (64, 3, 193, True, False), (176, 3, 63, False, False), (256, 1, 64, False, False),
                 (40, 3, 100, True, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("nstand,nchan,ntime,padded,conj", STORAGE_CASES)
def test_storage_fused(nstand, nchan, ntime, padded, conj):
    rng = np.random.default_rng(nstand * 1000 + ntime)
    x4 = full_range_ci4(rng, (ntime, nchan, 2 * nstand))
    la = LinAlg()
    views = []
    for x in (bf.ndarray(x4, dtype='ci4'), decoded_ci8(x4)):
        xv = bf.asarray(x, space='cuda').transpose((1, 0, 2))
        views.append(xv.conj() if conj else xv)
    got4, k4 = storage_call(la, views[0], nchan, nstand, padded)
    got8, k8 = storage_call(la, views[1], nchan, nstand, padded)
    assert k4 == [FUSED4], k4
    assert k8 == ['corr_storage_tc_kernel'], k8
    assert not np.isnan(got4).any()
    same_bits(got4, got8)
    same_bits(got4, storage_two_calls(la, views[0], nchan, nstand))
    if not conj:
        c = oracle_ci4(np.transpose(x4, (1, 0, 2)))
        same_bits(got4, ovis.to_storage(c.reshape(nchan, nstand, 2, nstand, 2)))


@pytest.mark.gpu
def test_storage_workspace_path():
    """nstand = 12: a 24 B station row, so the matrix correlator (SIMT) runs
    into the workspace, then the storage kernel; same bits as ci8."""
    rng = np.random.default_rng(12)
    nstand, nchan, ntime = 12, 3, 70
    x4 = full_range_ci4(rng, (ntime, nchan, 2 * nstand))
    la = LinAlg()
    got4, k4 = storage_call(la, bf.asarray(bf.ndarray(x4, dtype='ci4'), space='cuda').transpose((1, 0, 2)),
                            nchan, nstand, False)
    got8, _ = storage_call(la, bf.asarray(decoded_ci8(x4), space='cuda').transpose((1, 0, 2)), nchan, nstand, False)
    assert k4 == ['corr_simt_kernel', 'vis_to_storage_kernel'], k4
    same_bits(got4, got8)


# ------------------------------------------------------------- GPU: block
def volt_header(nchan, nstand, dtype, gulp):
    return {'_tensor': {'dtype': dtype, 'shape': [-1, nchan, nstand, 2],
                        'labels': ['time', 'freq', 'station', 'pol'],
                        'scales': [[0, 1 / 25e3], [50e6, 25e3], None, None],
                        'units': ['s', 'Hz', None, ['X', 'Y']]},
            'name': 'volts', 'gulp_nframe': gulp}


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


def run_pipeline(xs, hdr, nint, gulp, output):
    heads, outs = [], []
    with Pipeline() as p:
        src = blocks.copy(ArraysSource(xs, hdr, gulp), space='cuda')
        b = blocks.correlate(src, nint, output=output)
        blocks.callback_sink(b, lambda s: (heads.append(s.header), outs.append([])),
                             lambda s: outs[-1].append(np.array(s.data.copy('system'))))
        p.run()
    return heads, [np.concatenate(o, 0) for o in outs]


@pytest.mark.gpu
@pytest.mark.parametrize("output", ['matrix', 'storage'])
@pytest.mark.parametrize("nint,gulp", [(40, 40), (60, 20)])
def test_block_equals_the_ci8_pipeline(output, nint, gulp):
    """A ci4 ['time','freq','station','pol'] ring, two sequences, integrations
    of one gulp and of three: the same headers and output bytes as the same
    pipeline fed the decoded ci8."""
    rng = np.random.default_rng(nint + gulp)
    nchan, nstand = 3, 24
    x4s = [full_range_ci4(rng, (2 * nint, nchan, nstand, 2)), full_range_ci4(rng, (nint, nchan, nstand, 2))]
    got = {}
    for dtype in ('ci4', 'ci8'):
        xs = [bf.ndarray(x, dtype='ci4') for x in x4s] if dtype == 'ci4' else [decoded_ci8(x) for x in x4s]
        got[dtype] = run_pipeline(xs, volt_header(nchan, nstand, dtype, gulp), nint, gulp, output)
    (h4, o4), (h8, o8) = got['ci4'], got['ci8']
    assert len(h4) == 2 and h4 == h8
    assert [o.shape[0] for o in o4] == [2, 1]
    for a, b in zip(o4, o8):
        same_bits(a, b)


# ------------------------------------------------------ GPU: status codes
@pytest.mark.gpu
def test_ci4_correlate_status_codes():
    """bfLinAlgCorrelateCi4 takes ci4 and nothing else, one of a / b NULL;
    bfLinAlgMatMul keeps the reference's status for ci4."""
    h = LinAlg()

    def status(fn, a, b, c):
        return fn(h.obj, 1.0, None if a is None else a.as_BFarray(), None if b is None else b.as_BFarray(),
                  0.0, c.as_BFarray())
    x4, x8 = bf.zeros((8, 16), 'ci4', 'cuda'), bf.zeros((8, 16), 'ci8', 'cuda')
    c = bf.zeros((16, 16), 'cf32', 'cuda')
    ci4 = _bf.bfLinAlgCorrelateCi4
    assert status(_bf.bfLinAlgMatMul, None, x4, c) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    assert status(ci4, None, x4, c) == 0
    assert status(ci4, x4.transpose((1, 0)), None, c) == 0
    assert status(ci4, None, x8, c) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    assert status(ci4, x4, x4.transpose((1, 0)), c) == _bf.BF_STATUS_INVALID_ARGUMENT
    assert ci4(h.obj, 1.0, None, None, 0.0, c.as_BFarray()) == _bf.BF_STATUS_INVALID_ARGUMENT
    assert status(ci4, None, x4, bf.zeros((16, 32), 'cf32', 'cuda')[:, ::2]) == _bf.BF_STATUS_UNSUPPORTED_STRIDE
    assert status(ci4, None, x4, bf.zeros((16, 16), 'cf64', 'cuda')) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    assert status(ci4, None, bf.zeros((8, 16), 'ci4', 'system'), c) == _bf.BF_STATUS_UNSUPPORTED_SPACE
    assert status(ci4, None, bf.zeros((65536, 1, 1), 'ci4', 'cuda'), bf.zeros((65536, 1, 1), 'cf32', 'cuda')) == \
        _bf.BF_STATUS_UNSUPPORTED_SHAPE
    bf.device.stream_synchronize()


@pytest.mark.gpu
def test_ci4_storage_status_codes():
    """bfLinAlgCorrelateCi4ToStorage takes ci4 and nothing else, with
    bfLinAlgCorrelateToStorage's rejections; bfLinAlgCorrelateToStorage keeps
    its status for ci4."""
    h = LinAlg()

    def st(x, v, fn=_bf.bfLinAlgCorrelateCi4ToStorage):
        return fn(h.obj, x.as_BFarray(), v.as_BFarray())
    x = bf.zeros((3, 64, 8), 'ci4', 'cuda')
    v = bf.zeros((10, 3, 4), 'cf32', 'cuda')
    assert st(x, v) == 0
    assert st(x, v, _bf.bfLinAlgCorrelateToStorage) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    assert st(bf.zeros((3, 64, 8), 'ci8', 'cuda'), v) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    assert st(x, bf.zeros((10, 3, 4), 'cf64', 'cuda')) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    assert st(bf.zeros((3, 64, 8), 'ci4', 'system'), v) == _bf.BF_STATUS_UNSUPPORTED_SPACE
    assert st(bf.zeros((1, 3, 64, 8), 'ci4', 'cuda'), v) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(bf.zeros((3, 64, 7), 'ci4', 'cuda'), v) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(x, bf.zeros((9, 3, 4), 'cf32', 'cuda')) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(x, bf.zeros((10, 3, 8), 'cf32', 'cuda')[..., ::2]) == _bf.BF_STATUS_UNSUPPORTED_STRIDE
    raw = bf.zeros((3 * 64 * 8 + 10 * 3 * 4 * 8,), 'u8', 'cuda')
    xa, va = x.as_BFarray(), v.as_BFarray()
    xa.data = va.data = raw.as_BFarray().data
    assert _bf.bfLinAlgCorrelateCi4ToStorage(h.obj, xa, va) == _bf.BF_STATUS_INVALID_ARGUMENT
    bf.device.stream_synchronize()
