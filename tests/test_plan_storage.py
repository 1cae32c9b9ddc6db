"""The exec_storage protocol and handle statuses of the streaming plans
(bfPulseSearch*, bfSkFlag*, bfCoherentDedisp*, bfFold*), on the host: the
arrays claim cuda space but their data pointers are aligned dummies that are
never dereferenced, since no call here reaches a kernel.  The workspace sizes
are pinned so a change to a plan's layout shows up without a GPU."""
import ctypes

import pytest

from bifrost_b200.libbifrost import _bf, BFarray

S = _bf
DUMMY = 1 << 32            # 4096-aligned, never dereferenced
NBYTE = {'u8': 1, 'u16': 2, 'f32': 4, 'i32': 4, 'ci4': 1, 'ci8': 2, 'ci16': 4, 'cf32': 8}
DTYPE = {'u8': S.BF_DTYPE_U8, 'u16': S.BF_DTYPE_U16, 'f32': S.BF_DTYPE_F32, 'i32': S.BF_DTYPE_I32,
         'ci4': S.BF_DTYPE_CI4, 'ci8': S.BF_DTYPE_CI8, 'ci16': S.BF_DTYPE_CI16, 'cf32': S.BF_DTYPE_CF32}


def desc(dtype, shape):
    """A contiguous cuda-space BFarray descriptor at the dummy address."""
    a = BFarray()
    a.data = DUMMY
    a.space = S.BF_SPACE_CUDA
    a.dtype = DTYPE[dtype]
    a.ndim = len(shape)
    stride = NBYTE[dtype]
    for d in reversed(range(len(shape))):
        a.shape[d] = shape[d]
        a.strides[d] = stride
        stride *= shape[d]
    return a


def _ref(a):
    return None if a is None else ctypes.byref(a)


def pulse_search(widths, decim, shape):
    nblk = -(-(shape[-1] - max(widths) + 1) // decim)
    arr = (ctypes.c_int * len(widths))(*widths)
    arrays = [desc('f32', shape), desc('f32', list(shape[:-1]) + [nblk, 3])]
    return (S.bfPulseSearchCreate, lambda p: S.bfPulseSearchInit(p, len(widths), arr, decim),
            lambda p, ptr, size: S.bfPulseSearchExecute(p, *map(_ref, arrays), ptr, size),
            S.bfPulseSearchDestroy)


def sk_flag(window, dtype, shape, with_sk=False):
    nwin = -(-shape[-1] // window)
    arrays = [desc(dtype, shape), desc(dtype, shape),
              desc('f32', list(shape[:-1]) + [nwin]) if with_sk else None]
    return (S.bfSkFlagCreate, lambda p: S.bfSkFlagInit(p, window, 1, 1.0, 0.5, 1.5),
            lambda p, ptr, size: S.bfSkFlagExecute(p, *map(_ref, arrays), ptr, size),
            S.bfSkFlagDestroy)


def coherent_dedisp(nchan, f0, df, dm, nfft, dtype, shape):
    arrays = [desc(dtype, shape), desc('cf32', shape)]
    return (S.bfCoherentDedispCreate, lambda p: S.bfCoherentDedispInit(p, nchan, f0, df, dm, nfft),
            lambda p, ptr, size: S.bfCoherentDedispExecute(p, *map(_ref, arrays), ptr, size),
            S.bfCoherentDedispDestroy)


def fold(nbin, dtype, shape):
    nchan = shape[0]
    delays = (ctypes.c_double * nchan)(*[0.001 * c for c in range(nchan)])
    x, out, count = desc(dtype, shape), desc('f32', list(shape[:-1]) + [nbin]), desc('i32', [nchan, nbin])
    return (S.bfFoldCreate, lambda p: S.bfFoldInit(p, nbin, nchan, delays, 64e-6, 0.0, 1.4, 0.0, 0.0),
            lambda p, ptr, size: S.bfFoldExecute(p, ctypes.byref(x), 0, ctypes.byref(out), ctypes.byref(count),
                                                 0, ptr, size),
            S.bfFoldDestroy)


# (op, its arguments, workspace bytes of the (NULL, &size) query)
CASES = [
    ('sk_flag', (64, 'u8', [3, 4, 1000]), 1792),
    ('sk_flag', (256, 'f32', [2, 4096], True), 512),
    ('sk_flag', (2, 'u16', [5, 3, 7, 301]), 142848),
    ('pulse_search', ((1, 4, 16), 100, [2, 3, 1000]), 2816),
    ('pulse_search', ((1, 2, 4, 8), 256, [5, 4096]), 4864),
    ('pulse_search', ((3,), 1, [7, 50]), 4608),
    ('coherent_dedisp', (4, 1400., 1., 10., 1024, 'ci8', [4, 2, 5000]), 512),
    ('coherent_dedisp', (2, 800., -0.5, 3., 4096, 'cf32', [2, 3000]), 512),
    ('coherent_dedisp', (3, 1400., 1., 0., 256, 'ci4', [3, 1, 2, 100]), 512),
    ('fold', (64, 'u8', [4, 2, 5000]), 5376),
    ('fold', (1024, 'f32', [2, 100000]), 98560),
    ('fold', (7, 'u16', [3, 5, 7, 2000]), 6400),
]
OPS = {'pulse_search': pulse_search, 'sk_flag': sk_flag, 'coherent_dedisp': coherent_dedisp, 'fold': fold}


def _case_id(case):
    return '%s-%s' % (case[0], '-'.join(str(v).replace(' ', '') for v in case[1]))


@pytest.fixture(params=CASES, ids=[_case_id(c) for c in CASES])
def planned(request):
    op, args, size = request.param
    create, init, execute, destroy = OPS[op](*args)
    plan = ctypes.c_void_p()
    assert create(ctypes.byref(plan)) == S.BF_STATUS_SUCCESS
    assert init(plan) == S.BF_STATUS_SUCCESS
    yield plan, execute, size
    assert destroy(plan) == S.BF_STATUS_SUCCESS


def test_query_size(planned):
    plan, execute, size = planned
    got = S.BFsize(0)
    assert execute(plan, None, ctypes.byref(got)) == S.BF_STATUS_SUCCESS
    assert got.value == size


def test_caller_storage_too_small(planned):
    plan, execute, size = planned
    short = S.BFsize(size - 1)
    assert execute(plan, DUMMY, ctypes.byref(short)) == S.BF_STATUS_INSUFFICIENT_STORAGE


def test_pointer_without_size_is_refused(planned):
    plan, execute, _ = planned
    assert execute(plan, DUMMY, None) == S.BF_STATUS_INVALID_ARGUMENT


@pytest.mark.parametrize('op', sorted(OPS))
def test_handle_statuses(op):
    args = next(a for o, a, _ in CASES if o == op)
    create, _, execute, destroy = OPS[op](*args)
    size = S.BFsize(0)
    assert create(None) == S.BF_STATUS_INVALID_POINTER
    assert destroy(None) == S.BF_STATUS_INVALID_HANDLE
    assert execute(None, None, ctypes.byref(size)) == S.BF_STATUS_INVALID_HANDLE
    plan = ctypes.c_void_p()
    assert create(ctypes.byref(plan)) == S.BF_STATUS_SUCCESS
    assert plan.value
    assert execute(plan, None, ctypes.byref(size)) == S.BF_STATUS_INVALID_STATE
    assert destroy(plan) == S.BF_STATUS_SUCCESS
