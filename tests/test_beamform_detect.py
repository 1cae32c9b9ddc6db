"""Power beams in one pass: bfLinAlgBeamformDetect (LinAlg.beamform_detect),
beamform(..., detect=, nint=) and the block_scope(fuse=True) swap of
beamform -> detect -> reduce('time').

Every GPU case compares the call against its definition, the three calls
    bfLinAlgMatMul(1, w, x, 0, C) -> bfDetect(C as [.., nb/npb, npb, ntime]) -> bfReduce(sum)
on the uint32 view (so -0.0 != +0.0), against the oracle (oracle/beamform.py
beams, oracle/ops.py detect and reduce) within the fp32 error bound of the
sums, and asserts which kernels ran (tests/kernel_trace.py)."""
import os
import re
import subprocess

import numpy as np
import pytest

import bifrost_b200 as bf
from bifrost_b200 import blocks
from bifrost_b200.libbifrost import _bf
from bifrost_b200.linalg import LinAlg
from bifrost_b200.map import DETECT_MODES, detect as bf_detect
from bifrost_b200.pipeline import Pipeline
from oracle import beamform as obeamform
from oracle import ops as oops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CI4 = bf.DataType('ci4').as_numpy_dtype()
CI8 = bf.DataType('ci8').as_numpy_dtype()
CI16 = bf.DataType('ci16').as_numpy_dtype()
FUSED = 'beam_power_kernel'
NPB = {'scalar': 1, 'stokes': 2, 'stokes_i': 2, 'coherence': 2}
NPROD = {'scalar': 1, 'stokes': 4, 'stokes_i': 1, 'coherence': 4}


def volts(rng, shape, kind):
    """Voltages over the full range (-128 / -8 included) and their values."""
    lim = {'ci8': 128, 'ci4': 8, 'ci16': 32768}.get(kind, 128)
    re = rng.integers(-lim, lim, size=shape)
    im = rng.integers(-lim, lim, size=shape)
    re.flat[0], im.flat[-1] = -lim, -lim
    if kind == 'ci4':
        x = np.empty(shape, CI4)
        x['re_im'] = ((re & 0xF) << 4 | (im & 0xF)).astype(np.uint8)
    elif kind == 'cf32':
        x = (re + 1j * im).astype(np.complex64)
    else:
        x = np.empty(shape, CI8 if kind == 'ci8' else CI16)
        x['re'], x['im'] = re, im
    return x, re + 1j * im


def weights(rng, shape, kind, integer=False):
    if kind == 'ci16':
        w = np.empty(shape, CI16)
        w['re'] = rng.choice([-32767, 32767, -32768, 1, 0], size=shape)
        w['im'] = rng.integers(-32768, 32768, size=shape)
        return w, w['re'] + 1j * w['im'].astype(np.float64)
    if integer:
        lim = min(127, (2 ** 24 - 1) // (2 * 128 * shape[-1]))
        w = (rng.integers(-lim, lim + 1, size=shape) + 1j * rng.integers(-lim, lim + 1, size=shape))
    else:
        w = rng.normal(size=shape) + 1j * rng.normal(size=shape)
    w = w.astype(np.complex64)
    return w, w.astype(np.complex128)


def dev(a, kind=None):
    return bf.asarray(bf.ndarray(a, dtype='ci4') if kind == 'ci4' else a, space='cuda')


def kernels(fn):
    from kernel_trace import device_kernels
    return device_kernels(fn)


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def out_shape(bshape, nb, ntime, mode, nint):
    return tuple(bshape) + (nb // NPB[mode], NPROD[mode], ntime // nint)


def chain(d_w, d_x, mode, nint, oshape):
    """The definition: matmul -> detect -> reduce; returns (out, kernel names)."""
    nd = len(oshape)
    nb, ntime = oshape[nd - 3] * NPB[mode], oshape[nd - 1] * nint
    bshape = oshape[:nd - 3]
    res = {}

    def run():
        c = bf.zeros(bshape + (nb, ntime), 'cf32', 'cuda')
        LinAlg().matmul(1., d_w, d_x, 0., c)
        cv = c.reshape(bshape + (nb // NPB[mode], NPB[mode], ntime))
        d = bf.empty(bshape + (nb // NPB[mode], NPROD[mode], ntime), 'f32', 'cuda')
        bf_detect(cv, d, mode, nd - 2)
        if nint == 1:
            res['out'] = d
            return
        res['out'] = bf.empty(oshape, 'f32', 'cuda')
        bf.reduce(d, res['out'], 'sum')
    names = kernels(run)
    return np.asarray(res['out'].copy('system')), names


def fused(d_w, d_x, mode, nint, oshape, out=None):
    """LinAlg.beamform_detect into a fresh (or the given) out; returns (out, kernel names)."""
    d_out = bf.zeros(oshape, 'f32', 'cuda') if out is None else out
    names = kernels(lambda: LinAlg().beamform_detect(d_w, d_x, d_out, mode, nint))
    return np.asarray(d_out.copy('system')), names


def oracle(w, x, wv, xv, mode, nint, conj_w=False, conj_x=False):
    """[.., nb, K] x [.., K, ntime] -> [.., nb/npb, nprod, ntime/nint], and per
    output sum_t (F_x^2 + F_y^2) with F = sum_k |w_k| |x_k|, which bounds |b|."""
    if w.dtype.names:
        w = wv.astype(np.complex64)               # ci16 values are exact in cf32
    c = obeamform.matmul_ab(w, x, conj_a=conj_w, conj_b=conj_x)
    nd = c.ndim
    cv = c.reshape(c.shape[:nd - 2] + (c.shape[nd - 2] // NPB[mode], NPB[mode], c.shape[nd - 1]))
    d = oops.detect(cv, mode, nd - 1)
    out = d if nint == 1 else oops.reduce(d, nint, nd, 'sum')
    f = np.matmul(np.abs(wv), np.abs(xv)) ** 2
    f = f.reshape(cv.shape).sum(axis=nd - 1, keepdims=True)
    bound = f.reshape(f.shape[:nd] + (f.shape[nd] // nint, nint)).sum(-1)
    return out, np.broadcast_to(bound, out.shape)


def check(w, x, wv, xv, d_w, d_x, mode, nint, path='fused', conj_w=False, conj_x=False):
    """The call equals the chain bit for bit and the oracle within
    (nint + 8) 2^-23 + 8e-6 of sum |b|^2, and ran the expected kernels."""
    nd = d_x.ndim
    bshape = tuple(np.broadcast_shapes(d_w.shape[:nd - 2], d_x.shape[:nd - 2]))
    oshape = out_shape(bshape, d_w.shape[nd - 2], d_x.shape[nd - 1], mode, nint)
    want, cnames = chain(d_w, d_x, mode, nint, oshape)
    got, names = fused(d_w, d_x, mode, nint, oshape)
    if path == 'fused':
        assert len(names) == 1 and FUSED in names[0], names
    else:
        assert FUSED not in ''.join(names) and len(names) == len(cnames) and len(names) == (2 if nint == 1 else 3), \
            (names, cnames)
    assert got.shape == want.shape
    assert np.array_equal(u32(got), u32(want))
    ref, bound = oracle(w, x, wv, xv, mode, nint, conj_w, conj_x)
    err = np.abs(got.astype(np.float64) - ref.astype(np.float64))
    assert np.all(err <= ((nint + 8) * 2.0 ** -23 + 8e-6) * bound + 1e-30), err.max()
    return got


def case(rng, nb, K, ntime, nchan, xk, wk, mode, nint, integer=False, path='fused'):
    x, xv = volts(rng, (ntime, nchan, K), xk)
    w, wv = weights(rng, (nb, nchan, K), wk, integer)
    d_w = dev(w).transpose((1, 0, 2))
    d_x = dev(x, xk).transpose((1, 2, 0))
    return check(w.transpose(1, 0, 2), x.transpose(1, 2, 0), wv.transpose(1, 0, 2), xv.transpose(1, 2, 0),
                 d_w, d_x, mode, nint, path)


# ----------------------------------------------------------------- GPU: values
MODES = ['scalar', 'stokes', 'stokes_i', 'coherence']


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("xk", ['ci4', 'ci8'])
@pytest.mark.parametrize("wk", ['cf32', 'ci16'])
def test_modes_and_types(mode, xk, wk):
    """nb = 6 (not a multiple of the 8-beam tile), odd K, ntime not a multiple of 256."""
    rng = np.random.default_rng(MODES.index(mode) * 4 + 2 * (xk == 'ci4') + (wk == 'ci16'))
    case(rng, 6, 37, 816, 2, xk, wk, mode, 16)


NINTS = [(1, 300), (3, 771), (16, 4096), (256, 1280), (257, 771), (1000, 3000), (4000, 4000)]


@pytest.mark.gpu
@pytest.mark.parametrize("i,nint,ntime", [(i,) + v for i, v in enumerate(NINTS)])
def test_nint(i, nint, ntime):
    """Whole groups per CTA (nint <= 256), one group over several tiles (nint > 256), nint = ntime."""
    rng = np.random.default_rng(100 + i)
    mode = MODES[(i + 1) % 4]
    nb = [34, 2, 16, 6][i % 4] if mode != 'scalar' else [5, 1, 17][i % 3]
    case(rng, nb, [64, 130, 512][i % 3], ntime, 1 + i % 2, ['ci8', 'ci4'][i % 2], 'cf32', mode, nint)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ['stokes', 'scalar'])
def test_integer_weights(mode):
    """Integer-valued weights: every beam exact."""
    case(np.random.default_rng(7), 64, 512, 1024, 2, 'ci8', 'cf32', mode, 16, integer=True)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_zero_voltages(mode):
    """All-zero voltages: V = -2 (+0) = -0.0, and a sum started from 0.0 would give +0.0."""
    ntime, nchan, K, nb = 512, 2, 32, 4
    x = np.zeros((nchan, ntime, K), CI8)
    w = np.ones((nchan, nb, K), np.complex64)
    xt = x.transpose(0, 2, 1)
    got = check(w, xt, w, xt['re'] + 0j, dev(w), dev(x).transpose((0, 2, 1)), mode, 16)
    if mode == 'stokes':
        assert np.all(u32(got[:, :, 3]) == 0x80000000) and np.all(u32(got[:, :, :3]) == 0)


@pytest.mark.gpu
@pytest.mark.parametrize("xk", ['ci8', 'ci4'])
@pytest.mark.parametrize("conj_w,conj_x", [(True, False), (False, True)])
def test_conjugated_views(conj_w, conj_x, xk):
    rng = np.random.default_rng(8)
    x, xv = volts(rng, (300, 2, 40), xk)
    w, wv = weights(rng, (6, 2, 40), 'cf32')
    d_w, d_x = dev(w).transpose((1, 0, 2)), dev(x, xk).transpose((1, 2, 0))
    if conj_w:
        d_w = d_w.conj()
    if conj_x:
        d_x = d_x.conj()
    check(w.transpose(1, 0, 2), x.transpose(1, 2, 0), wv.transpose(1, 0, 2), xv.transpose(1, 2, 0),
          d_w, d_x, 'stokes', 4, conj_w=conj_w, conj_x=conj_x)


@pytest.mark.gpu
@pytest.mark.parametrize("xk", ['ci8', 'ci4'])
def test_misaligned_voltages_and_padded_out(xk):
    """A [..., 1:] voltage slice (any byte phase); out a padded view whose padding survives."""
    rng = np.random.default_rng(9)
    ntime, nchan, K, nb, nint = 700, 3, 77, 10, 7
    xbig, xvbig = volts(rng, (ntime, nchan, K + 1), xk)
    w, wv = weights(rng, (nb, nchan, K), 'cf32')
    d_w = dev(w).transpose((1, 0, 2))
    d_x = dev(xbig, xk)[..., 1:].transpose((1, 2, 0))
    got = check(w.transpose(1, 0, 2), xbig[..., 1:].transpose(1, 2, 0), wv.transpose(1, 0, 2),
                xvbig[..., 1:].transpose(1, 2, 0), d_w, d_x, 'coherence', nint)
    buf = np.full((nchan + 1, nb // 2 + 1, 6, ntime // nint + 3), -7.5, np.float32)
    d_buf = bf.asarray(buf, space='cuda')
    view = d_buf[:nchan, :nb // 2, 1:5, 2:2 + ntime // nint]
    padded, names = fused(d_w, d_x, 'coherence', nint, None, out=view)
    assert FUSED in names[0]
    full = np.asarray(d_buf.copy('system'))
    assert np.array_equal(u32(full[:nchan, :nb // 2, 1:5, 2:2 + ntime // nint]), u32(got))
    full[:nchan, :nb // 2, 1:5, 2:2 + ntime // nint] = -7.5
    assert np.all(full == -7.5)


@pytest.mark.gpu
def test_batch_dims_and_broadcast():
    """Two batch dims with padded strides, and weights broadcast over one of them."""
    rng = np.random.default_rng(10)
    nb, K, ntime = 8, 48, 512
    x, xv = volts(rng, (2, 3, K + 5, ntime), 'ci8')
    w, wv = weights(rng, (1, 3, nb, K), 'cf32')
    d_x = dev(x)[:, :, :K, :]
    # d_x has a K stride of ntime voltages, which only the workspace path takes;
    # d_xt is the same data with unit K stride and padded time / batch strides
    xt = np.ascontiguousarray(np.swapaxes(x, 2, 3))                      # [2, 3, ntime, K + 5]
    d_xt = dev(xt)[..., :K].transpose((0, 1, 3, 2))
    check(w, x[:, :, :K, :], wv, xv[:, :, :K, :], dev(w), d_xt, 'stokes_i', 16)
    check(w, x[:, :, :K, :], wv, xv[:, :, :K, :], dev(w), d_x, 'stokes_i', 16, path='workspace')


# ------------------------------------------------------- GPU: workspace path
@pytest.mark.gpu
@pytest.mark.parametrize("xk", ['ci16', 'cf32'])
@pytest.mark.parametrize("nint", [1, 16])
def test_workspace_voltage_types(xk, nint):
    case(np.random.default_rng(11), 6, 40, 320, 2, xk, 'cf32', 'stokes', nint, path='workspace')


@pytest.mark.gpu
def test_workspace_simt():
    os.environ['BFB_LINALG_SIMT'] = '1'
    try:
        case(np.random.default_rng(12), 6, 40, 320, 2, 'ci8', 'cf32', 'coherence', 8, path='workspace')
    finally:
        del os.environ['BFB_LINALG_SIMT']


# ----------------------------------------------------------- GPU: status codes
@pytest.mark.gpu
def test_status_codes_leave_out_untouched():
    h = LinAlg()
    w = bf.asarray(np.ones((2, 4, 8), np.complex64), space='cuda')
    x = bf.zeros((2, 8, 64), 'ci8', 'cuda')

    def st(out, mode=DETECT_MODES['stokes'], nint=16, w=w, x=x):
        before = np.asarray(out.copy('system')).tobytes()
        s = _bf.bfLinAlgBeamformDetect(h.obj, w.as_BFarray(), x.as_BFarray(), mode, nint, out.as_BFarray())
        if s != 0:
            assert np.asarray(out.copy('system')).tobytes() == before
        return s

    def o(shape, dtype='f32'):
        return bf.asarray(np.full(shape, 3.25, np.float32), space='cuda') if dtype == 'f32' else \
            bf.zeros(shape, dtype, 'cuda')
    good = (2, 2, 4, 4)
    assert st(o(good)) == 0
    assert st(o(good), mode=DETECT_MODES['jones']) == _bf.BF_STATUS_UNSUPPORTED
    assert st(o(good), mode=7) == _bf.BF_STATUS_UNSUPPORTED
    assert st(o(good), mode=-1) == _bf.BF_STATUS_UNSUPPORTED
    assert st(o(good), nint=0) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(o((2, 2, 4, 6)), nint=10) == _bf.BF_STATUS_INVALID_SHAPE          # 64 % 10
    odd = bf.asarray(np.ones((2, 3, 8), np.complex64), space='cuda')
    assert st(o((2, 1, 4, 4)), w=odd) == _bf.BF_STATUS_INVALID_SHAPE           # odd nb, polarised
    assert st(o((2, 3, 1, 4)), w=odd, mode=0) == 0                             # fine for scalar
    for shape in [(2, 2, 4, 3), (2, 2, 1, 4), (2, 4, 4, 4), (3, 2, 4, 4), (2, 4, 4)]:
        assert st(o(shape)) == _bf.BF_STATUS_INVALID_SHAPE, shape
    assert st(o(good, 'cf32')) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    assert st(o(good, 'f64')) == _bf.BF_STATUS_UNSUPPORTED_DTYPE
    # what bfLinAlgMatMul returns for the same w and x
    assert st(o(good), x=bf.zeros((2, 9, 64), 'ci8', 'cuda')) == _bf.BF_STATUS_INVALID_SHAPE
    assert st(o(good), x=bf.zeros((2, 8, 64), 'ci8', 'system')) == _bf.BF_STATUS_UNSUPPORTED_SPACE
    assert st(o(good), x=bf.zeros((2, 8, 64), 'u8', 'cuda')) == _bf.BF_STATUS_UNSUPPORTED_DTYPE


# ---------------------------------------------------------- GPU: ring pipelines
def volt_header(nchan, nstand, gulp, dtype='ci8'):
    return {'_tensor': {'dtype': dtype, 'shape': [-1, nchan, nstand, 2],
                        'labels': ['time', 'freq', 'station', 'pol'],
                        'scales': [[0, 1 / 25e3], [50e6, 25e3], None, None],
                        'units': ['s', 'Hz', None, ['X', 'Y']]},
            'name': 'volts', 'gulp_nframe': gulp}


def run_pipeline(x, hdr, w, mode, nint, how):
    """how: 'chain' (beamform -> detect -> reduce), 'fused' (beamform(detect=, nint=)),
    'fuse' (the chain under block_scope(fuse=True)).  Returns header, output, block kinds."""
    from bifrost_b200 import block_scope
    heads, outs = [], []
    with Pipeline() as p:
        src = blocks.copy(blocks.array_source(x, hdr, gulp_nframe=hdr['gulp_nframe']), space='cuda')
        if how == 'fused':
            b = blocks.beamform(src, w, detect=mode, nint=nint)
        else:
            with block_scope(fuse=(how == 'fuse')):
                b = blocks.reduce(blocks.detect(blocks.beamform(src, w), mode), 'time', nint)
        blocks.callback_sink(b, lambda s: heads.append(s.header),
                             lambda s: outs.append(np.array(s.data.copy('system'))))
        p.run()
    return heads, np.concatenate(outs, 0), [type(b).__name__ for b in p.blocks]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,nint,wdim", [('stokes', 16, 5), ('stokes_i', 4, 5), ('coherence', 32, 5),
                                            ('scalar', 8, 5), ('scalar', 16, 4), ('stokes', 8, 4)])
def test_pipelines_equal_the_chain(mode, nint, wdim):
    rng = np.random.default_rng(nint + wdim)
    nchan, nstand, gulp, ntime = 3, 12, 64, 320
    x, _ = volts(rng, (ntime, nchan, nstand, 2), 'ci8')
    wshape = (nchan, 5, 2, nstand, 2) if wdim == 5 else (nchan, 5, nstand, 2)
    w, _ = weights(rng, wshape, 'cf32')
    hdr = volt_header(nchan, nstand, gulp)
    ref_h, ref, kinds = run_pipeline(x, hdr, w, mode, nint, 'chain')
    assert 'DetectBlock' in kinds and 'ReduceBlock' in kinds
    assert ref.shape[0] == ntime // nint
    for how in ('fused', 'fuse'):
        h, got, kinds = run_pipeline(x, hdr, w, mode, nint, how)
        assert kinds.count('BeamformBlock') == 1 and 'DetectBlock' not in kinds and 'ReduceBlock' not in kinds
        assert h == ref_h
        assert np.array_equal(u32(got), u32(ref))


# ---------------------------------------------------------------- CPU: build
def test_kernels_compile_without_spills(tmp_path):
    """beam_power_kernel: 20 sm_90a instantiations, no spills, within the
    register budget of the beamformer's 2 (BT >= 4) or 3 (BT <= 2) CTAs per
    SM; beamform_kernel keeps its 20."""
    src = os.path.join(ROOT, 'bifrost_b200', 'csrc')
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    out = subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17',
                          '-I' + os.path.join(ROOT, 'include'), '-I' + src, '--expt-relaxed-constexpr',
                          '-Xptxas', '-v', '-c', os.path.join(src, 'beamform.cu'), '-o', str(tmp_path / 'b.o')],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    stats, entry = {}, None
    for line in out.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            entry = m.group(1)
            stats[entry] = ''
        elif entry:
            stats[entry] += line
    assert len([k for k in stats if 'beamform_kernel' in k]) == 20
    power = {k: v for k, v in stats.items() if FUSED in k}
    assert len(power) == 20, list(stats)
    for k, v in power.items():
        assert ' 0 bytes spill stores, 0 bytes spill loads' in v, (k, v)
        regs = int(re.search(r'Used (\d+) registers', v).group(1))
        smem = int(re.search(r'(\d+) bytes smem', v).group(1))
        bt = int(re.search(r'ELi(\d+)E', k).group(1))
        ncta = 3 if bt <= 2 else 2
        assert regs * 256 * ncta <= 65536 and smem * ncta <= 227 * 1024, (k, regs, smem)


# ------------------------------------------------------- CPU: block headers
class Seq(object):
    def __init__(self, header):
        self.header = header


def chain_header(hdr, w, mode, nint):
    """The header the three blocks give, from their own on_sequence."""
    with Pipeline():
        src = blocks.array_source(np.zeros((16, 4, 3, 2), CI8), hdr, gulp_nframe=16)
        b = blocks.beamform(src, w)
        d = blocks.detect(b, mode)
        r = blocks.reduce(d, 'time', nint)
    h = b.on_sequence(Seq(hdr))
    h.setdefault('gulp_nframe', hdr.get('gulp_nframe'))
    h = d.on_sequence(Seq(h))
    h.setdefault('gulp_nframe', hdr.get('gulp_nframe'))
    return r.on_sequence(Seq(h))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("wdim", [4, 5])
@pytest.mark.parametrize("nint,gulp", [(4, 16), (16, 16), (8, None)])
def test_block_header_equals_the_chain(mode, wdim, nint, gulp):
    hdr = volt_header(4, 3, gulp)
    if gulp is None:
        del hdr['gulp_nframe']
    w = np.ones((4, 5, 2, 3, 2) if wdim == 5 else (4, 5, 3, 2), np.complex64)
    want = chain_header(hdr, w, mode, nint)
    with Pipeline():
        src = blocks.array_source(np.zeros((16, 4, 3, 2), CI8), hdr, gulp_nframe=16)
        b = blocks.beamform(src, w, detect=mode, nint=nint, gulp_nframe=16)
    got = b.on_sequence(Seq(hdr))
    assert got == want
    t = got['_tensor']
    assert t['dtype'] == 'f32' and t['scales'][0] == [0, nint / 25e3]
    if wdim == 5:
        assert t['labels'] == ['time', 'freq', 'beam', 'pol']
        assert t['shape'] == [-1, 4, 5, 2 if mode == 'scalar' else NPROD[mode]]
    else:
        assert t['labels'] == ['time', 'freq', 'beam'] and t['shape'] == [-1, 4, 5]


def test_block_rejects_bad_arguments():
    w5 = np.ones((4, 5, 2, 3, 2), np.complex64)
    with Pipeline():
        src = blocks.array_source(np.zeros((16, 4, 3, 2), CI8), volt_header(4, 3, 16), gulp_nframe=16)
        for kw in [dict(detect='jones'), dict(detect='stokes', nint=0), dict(nint=4), dict(detect='x')]:
            with pytest.raises(ValueError):
                blocks.beamform(src, w5, **kw)
        with pytest.raises(ValueError):
            blocks.beamform(src, np.ones((4, 5, 3, 3, 2), np.complex64))
        b = blocks.beamform(src, w5, detect='stokes', nint=6)
    with pytest.raises(ValueError):                  # gulp 16 is not a multiple of 6
        b.on_sequence(Seq(volt_header(4, 3, 16)))


# ---------------------------------------------------------- CPU: fuse matcher
def build_chain(mode='stokes', axis='time', factor=8, op='sum', fuse=(True, True, True), branch=False,
                daxis=None):
    from bifrost_b200 import block_scope
    w5 = np.ones((4, 5, 2, 3, 2), np.complex64)
    with Pipeline() as p:
        src = blocks.array_source(np.zeros((16, 4, 3, 2), CI8), volt_header(4, 3, 16), gulp_nframe=16)
        with block_scope(fuse=fuse[0], gpu=0, core=1):
            b = blocks.beamform(src, w5, gulp_nframe=16)
        with block_scope(fuse=fuse[1]):
            d = blocks.detect(b, mode, daxis)
        with block_scope(fuse=fuse[2]):
            r = blocks.reduce(d, axis, factor, op)
        if branch:
            blocks.callback_sink(d)
        sink = blocks.callback_sink(r)
    return p, src, sink


def test_fuse_swaps_beamform_detect_reduce():
    from bifrost_b200.blocks.beamform import BeamformBlock
    p, src, sink = build_chain()
    p._fuse_chains()
    kinds = [type(b).__name__ for b in p.blocks]
    assert 'DetectBlock' not in kinds and 'ReduceBlock' not in kinds and kinds.count('BeamformBlock') == 1
    bm = [b for b in p.blocks if isinstance(b, BeamformBlock)][0]
    assert (bm.detect, bm.nint, bm.gulp_nframe, bm.gpu, bm.core) == ('stokes', 8, 16, 0, 1)
    assert src.orings[0].consumers == [bm] and bm.orings[0].consumers == [sink] and bm.orings[0].owner is bm


@pytest.mark.parametrize("kw", [dict(op='mean'), dict(axis='freq', factor=2), dict(mode='jones'),
                                dict(branch=True), dict(fuse=(True, False, True)), dict(fuse=(False, True, True)),
                                dict(fuse=(True, True, False)), dict(daxis='beam')])
def test_fuse_leaves_other_chains_alone(kw):
    p, src, sink = build_chain(**kw)
    before = list(p.blocks)
    p._fuse_chains()
    assert p.blocks == before
