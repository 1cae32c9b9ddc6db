"""Edges of bfFft (csrc/fft.cu): every kernel that run_pass / run_axis can
pick, at the shapes, strides, element kinds and line counts where each one
has its own code.

Every test reads the kernels a call ran from torch.profiler (kernel_trace.py)
and checks their names with the template arguments.  The element kind of the
fast kernels is the FftInKind value: FK_CF32 = 0, FK_CI8 = 1, FK_CI16 = 2.  A
change in the dispatch therefore cannot move a case onto another kernel
unnoticed.  Values are compared with oracle/fft.py in fp64:
max |err| <= 1e-5 rms(gold), and 1e-12 rms(gold) for fp64 transforms.

__global__ in fft.cu                      test that asserts it ran
fft4096_fast_kernel<0|1|2>                test_fast_kernels, test_line_counts,
                                          test_padded_and_negative_batch_strides,
                                          test_in_place_one_axis, test_guppi_layout_fftshift
fft_fast_kernel<0|1|2, R3 = 1..8>         test_fast_kernels, test_line_counts,
                                          test_strided_output, test_in_place_2d
fft_fast_kernel<0|1|2, 16>                test_strided_output (n = 4096, strided store),
                                          test_four_step_pass_a_on_registers (pass B)
fft_regs_kernel<0|1|2, 16|32>             test_four_step_pass_a_on_registers
fft_pass_kernel<float>, Stockham          test_reversed_input_axis, test_ci4_on_the_generic_kernel,
                                          test_r2c_unsigned, test_four_step_generic_pass_a,
                                          test_in_place_2d
fft_pass_kernel<float>, direct DFT        test_direct_dft, test_r2c_unsigned (n = 1000)
fft_pass_kernel<double>                   test_fp64_c2c, test_real_long_fix_kernels
bluestein_{pre,mul,post}_kernel<float>    test_bluestein
bluestein_{pre,mul,post}_kernel<double>   test_fp64_c2c (n = 10000)
fft_r2c_fix_kernel<float|double>          test_real_long_fix_kernels
fft_c2r_fix_kernel<float|double>          test_real_long_fix_kernels

The fused spectrometer (spectrometer_kernel<F>, spectrometer.cu) shares
fft4096.cuh with fft4096_fast_kernel; its input and output layouts are tested
at the end against the same fp64 chain as tests/test_spectrometer.py."""
import re

import numpy as np
import pytest

import bifrost_b200 as bf
from bifrost_b200.fft import Fft
from kernel_trace import device_kernels
from oracle import fft as offt
from test_spectrometer import close, oracle_chain

pytestmark = pytest.mark.gpu

CI4 = bf.DataType('ci4').as_numpy_dtype()
CI8 = bf.DataType('ci8').as_numpy_dtype()
CI16 = bf.DataType('ci16').as_numpy_dtype()
FK = {'cf32': 0, 'ci8': 1, 'ci16': 2}           # FftInKind: template argument of the fast kernels
FAST_N = [256, 512, 1024, 2048, 4096]           # R3 = n / 256 = 1, 2, 4, 8, 16
DIRECTIONS = [(False, False), (False, True), (True, False), (True, True)]    # (inverse, fftshift)


# ------------------------------------------------------------------ helpers
def short(name):
    """'void bfb::fft_fast_kernel<1, 4>(bfb::FftPass<float>)' -> 'fft_fast_kernel<1, 4>'"""
    m = re.search(r'(\w+(?:<[^()]*>)?)\(', name)
    return m.group(1) if m else name


def compare(got, gold, tol=1e-5):
    gold = np.asarray(gold)
    rms = np.sqrt(np.mean(np.abs(gold) ** 2))
    err = np.abs(np.asarray(got) - gold).max()
    assert err <= tol * rms, "max|err| / rms(gold) = %.3g > %g" % (err / rms, tol)


def host(d):
    return np.asarray(d.copy('system'))


def signal(kind, shape, rng):
    """An input of `kind` and the complex128 values the kernels read from it
    (integer kinds scaled as on load).  Integers are uniform over their full
    range, and the most negative value (-8, -128, -32768) is forced into
    scattered samples, in both parts of some of them.  (The positions are
    random: a periodic pattern would put spectral lines far above the rms.)"""
    if kind in ('cf32', 'cf64'):
        x = rng.normal(size=shape) + 1j * rng.normal(size=shape)
        x = x.astype(np.complex64 if kind == 'cf32' else np.complex128)
        return x, x.astype(np.complex128)
    lim = {'ci4': 8, 'ci8': 128, 'ci16': 32768}[kind]
    re_ = rng.integers(-lim, lim, size=shape)
    im_ = rng.integers(-lim, lim, size=shape)
    size = int(np.prod(shape))
    at = rng.choice(size, size=max(8, size // 1024), replace=False)
    re_.reshape(-1)[at] = -lim
    im_.reshape(-1)[at[::2]] = -lim
    if kind == 'ci4':
        x = np.zeros(shape, CI4)
        x['re_im'] = ((re_ & 0xF) << 4 | (im_ & 0xF)).astype(np.uint8)
        return x, offt.to_complex128(x, 'ci4') * offt.SCALE['ci4']
    x = np.empty(shape, CI8 if kind == 'ci8' else CI16)
    x['re'], x['im'] = re_, im_
    return x, offt.to_complex128(x, kind) * offt.SCALE[kind]


def execute(d_in, d_out, axes, inverse=False, fftshift=False, reset=None):
    """One planned bfFftExecute; returns the kernels it ran, short names, in order."""
    plan = Fft()
    plan.init(d_in, d_out, axes=axes, apply_fftshift=fftshift)
    return [short(k) for k in device_kernels(lambda: plan.execute(d_in, d_out, inverse), reset=reset)]


def fast_kernel(kind, n):
    """The kernel a unit-stride c2c line of n = 256..4096 points runs on."""
    if n == 4096:
        return 'fft4096_fast_kernel<%d>' % FK[kind]
    return 'fft_fast_kernel<%d, %d>' % (FK[kind], n // 256)


def filled(shape, dtype=np.complex64):
    """A recognisable fill for the parts of an output array a call must not write."""
    v = 1234.5 - 678.25j if np.dtype(dtype).kind == 'c' else 1234.5
    return np.full(shape, v, dtype)


# ------------------------------------------------------------- fast kernels
@pytest.mark.parametrize("kind", ['cf32', 'ci8', 'ci16'])
@pytest.mark.parametrize("n", FAST_N)
def test_fast_kernels(kind, n):
    """Each kind and R3 of fft_fast_kernel and fft4096_fast_kernel, both
    directions, with and without fftshift.  Two full CTAs of 4096 / n lines
    and a partial third."""
    lines = 2 * (4096 // n) + 3
    x, xv = signal(kind, (lines, n), np.random.default_rng(n + FK[kind]))
    d_x = bf.asarray(x, space='cuda')
    d_y = bf.empty((lines, n), dtype='cf32', space='cuda')
    for inverse, shift in DIRECTIONS:
        assert execute(d_x, d_y, [1], inverse, shift) == [fast_kernel(kind, n)]
        compare(host(d_y), offt.fft(xv, [1], inverse=inverse, fftshift=shift))


@pytest.mark.parametrize("kind,n,lines", [
    ('cf32', 256, 7),                  # 16 lines per CTA: one partial CTA
    ('ci8', 1024, 5),                  # 4 lines per CTA: one full, one partial
    ('ci16', 4096, 2368 + 45),         # past the grid cap of 148 x 16 CTAs
    ('ci8', 256, 2368 * 16 + 21)])     # past the cap, with a partial last group
def test_line_counts(kind, n, lines):
    """Idle line slots of a partial CTA, and the grid-stride loop past the
    grid cap.  The output is all but the last row of a larger array: the row
    after it must stay untouched."""
    x, xv = signal(kind, (lines, n), np.random.default_rng(lines))
    d_x = bf.asarray(x, space='cuda')
    d_base = bf.asarray(filled((lines + 1, n)), space='cuda')
    d_y = d_base[:lines]
    for inverse, shift in ((False, True), (True, False)):
        assert execute(d_x, d_y, [1], inverse, shift) == [fast_kernel(kind, n)]
        got = host(d_base)
        compare(got[:lines], offt.fft(xv, [1], inverse=inverse, fftshift=shift))
        np.testing.assert_array_equal(got[lines], filled(n))


@pytest.mark.parametrize("kind", ['cf32', 'ci8', 'ci16'])
@pytest.mark.parametrize("n", FAST_N)
def test_strided_output(kind, n):
    """Output axis stride of 16 bytes (every other cf32 of a wider array):
    fft_fast_kernel's strided store.  n = 4096 goes there too, not to
    fft4096_fast_kernel.  The slots in between stay untouched."""
    lines = 4096 // n + 1
    x, xv = signal(kind, (lines, n), np.random.default_rng(10 * n + FK[kind]))
    d_x = bf.asarray(x, space='cuda')
    d_base = bf.asarray(filled((lines, 2 * n)), space='cuda')
    d_y = d_base[:, ::2]
    for inverse, shift in DIRECTIONS:
        assert execute(d_x, d_y, [1], inverse, shift) == ['fft_fast_kernel<%d, %d>' % (FK[kind], n // 256)]
        got = host(d_base)
        compare(got[:, ::2], offt.fft(xv, [1], inverse=inverse, fftshift=shift))
        np.testing.assert_array_equal(got[:, 1::2], filled((lines, n)))


@pytest.mark.parametrize("kind", ['cf32', 'ci8'])
@pytest.mark.parametrize("n", [1024, 4096])
def test_padded_and_negative_batch_strides(kind, n):
    """Two batch dims with padded strides and an offset base pointer, then the
    same with both batch dims reversed on the input and the outer one on the
    output.  Padding of the output stays untouched."""
    rng = np.random.default_rng(n + 7)
    base, bv = signal(kind, (3, 7, n + 16), rng)
    d_base = bf.asarray(base, space='cuda')
    views = [(np.s_[:, 1:6, 8:8 + n], np.s_[:, :5, :n]),
             (np.s_[::-1, 5:0:-1, 8:8 + n], np.s_[::-1, :5, :n])]
    for iv, ov in views:
        d_obase = bf.asarray(filled((3, 6, n + 8)), space='cuda')
        d_x, d_y = d_base[iv], d_obase[ov]
        for inverse, shift in ((False, True), (True, True)):
            assert execute(d_x, d_y, [2], inverse, shift) == [fast_kernel(kind, n)]
            got = host(d_obase)
            compare(got[ov], offt.fft(bv[iv], [2], inverse=inverse, fftshift=shift))
            pad = np.ones(got.shape, bool)
            pad[ov] = False
            np.testing.assert_array_equal(got[pad], filled(int(pad.sum())))


@pytest.mark.parametrize("kind", ['cf32', 'ci8', 'ci16'])
@pytest.mark.parametrize("n", FAST_N)
def test_reversed_input_axis(kind, n):
    """x[:, ::-1] has an axis stride of minus one element.  The fast kernels
    index a line forward from its first element, so such a view must take
    fft_pass_kernel.  The view is the first half of each row of a
    (lines, 2n) array read backwards: a kernel that walked forward instead
    would still read inside the row, and the test fails on values."""
    lines = 3
    base, bv = signal(kind, (lines, 2 * n), np.random.default_rng(20 * n + FK[kind]))
    d_base = bf.asarray(base, space='cuda')
    d_x = d_base[:, n - 1::-1]
    assert d_x.strides[1] < 0
    xv = bv[:, n - 1::-1]
    d_y = bf.empty((lines, n), dtype='cf32', space='cuda')
    for inverse, shift in DIRECTIONS:
        names = execute(d_x, d_y, [1], inverse, shift)
        compare(host(d_y), offt.fft(xv, [1], inverse=inverse, fftshift=shift))
        assert names == ['fft_pass_kernel<float>']


@pytest.mark.parametrize("n", [1024, 4096])
def test_in_place_one_axis(n):
    rng = np.random.default_rng(n + 3)
    x, xv = signal('cf32', (9, n), rng)
    d_x = bf.asarray(x, space='cuda')

    def reset():
        d_x[...] = x
    for inverse, shift in ((False, True), (True, True)):
        assert execute(d_x, d_x, [1], inverse, shift, reset=reset) == [fast_kernel('cf32', n)]
        compare(host(d_x), offt.fft(xv, [1], inverse=inverse, fftshift=shift))


def test_in_place_2d():
    """Axis 1 on the fast kernel, then axis 0 (strided) on the generic one,
    both in place."""
    x, xv = signal('cf32', (256, 512), np.random.default_rng(33))
    d_x = bf.asarray(x, space='cuda')

    def reset():
        d_x[...] = x
    for inverse, shift in DIRECTIONS:
        names = execute(d_x, d_x, [0, 1], inverse, shift, reset=reset)
        assert names == ['fft_fast_kernel<0, 2>', 'fft_pass_kernel<float>']
        compare(host(d_x), offt.fft(xv, [0, 1], inverse=inverse, fftshift=shift))


# ----------------------------------------------------------------- four-step
@pytest.mark.parametrize("kind", ['cf32', 'ci8', 'ci16'])
@pytest.mark.parametrize("n", [8192, 1 << 14, 1 << 16, 1 << 17])
def test_four_step_pass_a_on_registers(kind, n):
    """n = n1 * n2 with n2 = min(4096, n / 16): pass A (n1 = 16 or 32, strided,
    inter-pass twiddle, fftshift as a sign or a rotation) on fft_regs_kernel,
    pass B on fft_fast_kernel with a strided store."""
    n2 = min(4096, n // 16)
    n1 = n // n2
    want = ['fft_regs_kernel<%d, %d>' % (FK[kind], n1), 'fft_fast_kernel<0, %d>' % (n2 // 256)]
    x, xv = signal(kind, (3, n), np.random.default_rng(n + FK[kind]))
    d_x = bf.asarray(x, space='cuda')
    d_y = bf.empty((3, n), dtype='cf32', space='cuda')
    for inverse, shift in DIRECTIONS:
        assert execute(d_x, d_y, [1], inverse, shift) == want
        compare(host(d_y), offt.fft(xv, [1], inverse=inverse, fftshift=shift))


def test_four_step_generic_pass_a():
    """n = 2^20 = 256 x 4096: pass A (n1 = 256) on fft_pass_kernel."""
    n = 1 << 20
    x, xv = signal('cf32', (2, n), np.random.default_rng(20))
    d_x = bf.asarray(x, space='cuda')
    d_y = bf.empty((2, n), dtype='cf32', space='cuda')
    for inverse, shift in ((False, True), (True, True)):
        assert execute(d_x, d_y, [1], inverse, shift) == ['fft_pass_kernel<float>', 'fft_fast_kernel<0, 16>']
        compare(host(d_y), offt.fft(xv, [1], inverse=inverse, fftshift=shift))


# ------------------------------------------------- lengths that are not pow2
@pytest.mark.parametrize("n", [1001, 4095, 6000, 8191])
def test_direct_dft(n):
    """Direct DFT of fft_pass_kernel up to the one-pass limit (8191 is prime):
    c2c both ways with fftshift (odd n: the phase ramp), r2c and c2r.  Its
    sums run over n terms and are kept in double."""
    rng = np.random.default_rng(n)
    lines = 6
    x, xv = signal('cf32', (lines, n), rng)
    d_x = bf.asarray(x, space='cuda')
    d_y = bf.empty((lines, n), dtype='cf32', space='cuda')
    for inverse, shift in DIRECTIONS:
        assert execute(d_x, d_y, [1], inverse, shift) == ['fft_pass_kernel<float>']
        compare(host(d_y), offt.fft(xv, [1], inverse=inverse, fftshift=shift))
    # r2c
    r = rng.normal(size=(lines, n)).astype(np.float32)
    d_r = bf.asarray(r, space='cuda')
    d_s = bf.empty((lines, n // 2 + 1), dtype='cf32', space='cuda')
    assert execute(d_r, d_s, [1]) == ['fft_pass_kernel<float>']
    compare(host(d_s), offt.fft(r.astype(np.float64), [1]))
    # c2r of a Hermitian half-spectrum
    spec = np.fft.rfft(r.astype(np.float64), axis=1).astype(np.complex64)
    d_spec = bf.asarray(spec, space='cuda')
    d_back = bf.empty((lines, n), dtype='f32', space='cuda')
    assert execute(d_spec, d_back, [1]) == ['fft_pass_kernel<float>']
    compare(host(d_back), offt.fft(spec.astype(np.complex128), [1], real_out_len=n))


@pytest.mark.parametrize("kind,n", [('cf32', 8193), ('ci16', 12289), ('ci4', 9001)])
def test_bluestein(kind, n):
    """n > 8192, not a power of two: chirp-z on the m = 32768 four-step
    transforms (pass A on registers, pass B on the fast kernel)."""
    x, xv = signal(kind, (3, n), np.random.default_rng(n))
    d_x = bf.asarray(x, space='cuda')
    d_y = bf.empty((3, n), dtype='cf32', space='cuda')
    want = {'bluestein_pre_kernel<float>', 'bluestein_mul_kernel<float>', 'bluestein_post_kernel<float>',
            'fft_regs_kernel<0, 16>', 'fft_fast_kernel<0, 8>'}
    for inverse, shift in DIRECTIONS:
        names = execute(d_x, d_y, [1], inverse, shift)
        assert set(names) == want, names
        assert names[-1] == 'bluestein_post_kernel<float>', names
        compare(host(d_y), offt.fft(xv, [1], inverse=inverse, fftshift=shift))


# ------------------------------------------------------------ integer inputs
@pytest.mark.parametrize("n", [256, 4096])
def test_ci4_on_the_generic_kernel(n):
    """ci4 (high nibble real) with -8 in both nibbles: never a fast kernel."""
    x, xv = signal('ci4', (5, n), np.random.default_rng(n + 4))
    d_x = bf.asarray(x, space='cuda')
    d_y = bf.empty((5, n), dtype='cf32', space='cuda')
    for inverse, shift in DIRECTIONS:
        assert execute(d_x, d_y, [1], inverse, shift) == ['fft_pass_kernel<float>']
        compare(host(d_y), offt.fft(xv, [1], inverse=inverse, fftshift=shift))


@pytest.mark.parametrize("dtype,bf_dtype", [(np.uint8, 'u8'), (np.uint16, 'u16')])
@pytest.mark.parametrize("n", [512, 1000])
def test_r2c_unsigned(dtype, bf_dtype, n):
    """u8 / u16 real inputs, scaled by 1/256 and 1/65536 on load, over their
    full range (0 and the maximum forced in)."""
    top = np.iinfo(dtype).max
    x = np.random.default_rng(n).integers(0, top + 1, size=(6, n)).astype(dtype)
    x[:, 0], x[:, 1], x[2] = top, 0, top
    d_x = bf.asarray(x, space='cuda')
    d_y = bf.empty((6, n // 2 + 1), dtype='cf32', space='cuda')
    assert execute(d_x, d_y, [1]) == ['fft_pass_kernel<float>']
    compare(host(d_y), offt.fft(x.astype(np.float64) * offt.SCALE[bf_dtype], [1]))


def test_guppi_layout_fftshift():
    """The unfused GUPPI chain's transform: ci8 [frame, pol, chan, 4096] over
    the last axis with fftshift, 320 lines."""
    x, xv = signal('ci8', (4, 2, 40, 4096), np.random.default_rng(4096))
    d_x = bf.asarray(x, space='cuda')
    d_y = bf.empty(x.shape, dtype='cf32', space='cuda')
    assert execute(d_x, d_y, [3], False, True) == ['fft4096_fast_kernel<1>']
    compare(host(d_y), offt.fft(xv, [3], fftshift=True))


# ---------------------------------------------------------------------- fp64
@pytest.mark.parametrize("n", [16, 1001, 4096, 8192, 1 << 14, 10000])
def test_fp64_c2c(n):
    """cf64: Stockham up to 8192 in one pass, the direct DFT, four-step 2^14
    on the generic kernel both passes, Bluestein<double> at 10000."""
    x, xv = signal('cf64', (3, n), np.random.default_rng(n + 64))
    d_x = bf.asarray(x, space='cuda')
    d_y = bf.empty((3, n), dtype='cf64', space='cuda')
    if n == 10000:
        want = {'bluestein_pre_kernel<double>', 'bluestein_mul_kernel<double>',
                'bluestein_post_kernel<double>', 'fft_pass_kernel<double>'}
    else:
        want = {'fft_pass_kernel<double>'}
    npass = 2 if n == 1 << 14 else 1
    for inverse, shift in DIRECTIONS:
        names = execute(d_x, d_y, [1], inverse, shift)
        assert set(names) == want, names
        if n != 10000:
            assert len(names) == npass, names
        compare(host(d_y), offt.fft(xv, [1], inverse=inverse, fftshift=shift), tol=1e-12)


@pytest.mark.parametrize("prec", ['float', 'double'])
def test_real_long_fix_kernels(prec):
    """r2c and c2r at n = 2^14: one complex transform of n / 2 = 8192 points and
    the O(n) fix-up kernel (8192 splits into 16 x 512 in fp32 only)."""
    n, lines = 1 << 14, 3
    fp64 = prec == 'double'
    rdt, cdt = (np.float64, np.complex128) if fp64 else (np.float32, np.complex64)
    half = ['fft_pass_kernel<double>'] if fp64 else ['fft_regs_kernel<0, 16>', 'fft_fast_kernel<0, 2>']
    tol = 1e-12 if fp64 else 1e-5
    x = np.random.default_rng(14).normal(size=(lines, n)).astype(rdt)
    d_x = bf.asarray(x, space='cuda')
    d_s = bf.empty((lines, n // 2 + 1), dtype='cf64' if fp64 else 'cf32', space='cuda')
    assert execute(d_x, d_s, [1]) == half + ['fft_r2c_fix_kernel<%s>' % prec]
    compare(host(d_s), offt.fft(x.astype(np.float64), [1]), tol=tol)
    spec = np.fft.rfft(x.astype(np.float64), axis=1).astype(cdt)
    d_spec = bf.asarray(spec, space='cuda')
    d_back = bf.empty((lines, n), dtype='f64' if fp64 else 'f32', space='cuda')
    assert execute(d_spec, d_back, [1]) == ['fft_c2r_fix_kernel<%s>' % prec] + half
    compare(host(d_back), offt.fft(spec.astype(np.complex128), [1], real_out_len=n), tol=tol)


# -------------------------------------------------------- fused spectrometer
def voltages(shape, rng):
    """Full-range ci8 [.., nfft, pol] as signal() makes it, -128 included."""
    x, _ = signal('ci8', shape, rng)
    return x


def spectrometer_dev(d_x, d_o, f_avg, beta=0.0):
    """Runs the fused spectrometer on the device; asserts it took spectrometer_kernel<f_avg>."""
    reset = None
    if beta != 0:                                 # the result depends on the output: restore it
        o0 = host(d_o)

        def reset():
            d_o[...] = o0
    names = device_kernels(lambda: bf.spectrometer(d_x, d_o, 4096, f_avg, beta), reset=reset)
    assert [short(k) for k in names] == ['spectrometer_kernel<%d>' % f_avg]


def test_spectrometer_one_frame_3d_input():
    """[chan, nfft, pol]: one frame without a frame dim."""
    x = voltages((5, 4096, 2), np.random.default_rng(1))
    d_o = bf.asarray(np.full((4, 5 * 4096 // 8), np.nan, np.float32), space='cuda')
    spectrometer_dev(bf.asarray(x, space='cuda'), d_o, 8)
    close(host(d_o), oracle_chain(x[None], 8))


def test_spectrometer_padded_input_strides():
    """A ring span's view: padded channel stride (4096 + 32 samples) and frame
    stride (7 channels), and a base pointer inside the allocation."""
    base = voltages((3, 7, 4096 + 32, 2), np.random.default_rng(2))
    view = np.s_[:, 1:6, 16:16 + 4096, :]
    d_x = bf.asarray(base, space='cuda')[view]
    assert d_x.strides[1] == (4096 + 32) * 4 and d_x.strides[0] == 7 * d_x.strides[1]
    d_o = bf.asarray(np.full((4, 5 * 4096 // 4), np.nan, np.float32), space='cuda')
    spectrometer_dev(d_x, d_o, 4)
    close(host(d_o), oracle_chain(base[view], 4))


def test_spectrometer_padded_output():
    """Output [1, 4, nchan nfft / f]: a leading unit dim and a Stokes stride
    padded by 64 floats, which stay untouched."""
    x = voltages((2, 3, 4096, 2), np.random.default_rng(3))
    w = 3 * 4096 // 16
    d_base = bf.asarray(filled((1, 4, w + 64), np.float32), space='cuda')
    spectrometer_dev(bf.asarray(x, space='cuda'), d_base[:, :, :w], 16)
    got = host(d_base)
    close(got[0, :, :w], oracle_chain(x, 16))
    np.testing.assert_array_equal(got[0, :, w:], filled((4, 64), np.float32))


@pytest.mark.parametrize("f_avg", [2, 32])
def test_spectrometer_beta_half(f_avg):
    """out = 0.5 out + the new gulp, from an out of the same magnitude."""
    rng = np.random.default_rng(4 + f_avg)
    x0, x = voltages((2, 4, 4096, 2), rng), voltages((2, 4, 4096, 2), rng)
    o0 = oracle_chain(x0, f_avg).astype(np.float32)
    d_o = bf.asarray(o0, space='cuda')
    spectrometer_dev(bf.asarray(x, space='cuda'), d_o, f_avg, beta=0.5)
    close(host(d_o), 0.5 * o0.astype(np.float64) + oracle_chain(x, f_avg))
