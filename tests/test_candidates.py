"""bfCandidates*: friends-of-friends clustering of peak maps into candidates.

CPU: the oracle (oracle/candidates.py) against a brute-force O(n^2) search of
the friendship graph and on edge cases, the pulse_search header key the sink
needs, the sink's header checks and line format, Init refusals and the
descriptor-only statuses of Execute.  GPU: bfCandidatesExecute bit for bit
against the oracle on random, chained, lattice, dense, overflowing and
strided maps, repeatability, the workspace modes, a fixed kernel list, and a
filterbank through fdmt -> pulse_search -> write_candidates."""
import ctypes
import os
import sys
from collections import deque
from copy import deepcopy

import numpy as np
import pytest

import bifrost_b200 as bf
from bifrost_b200.libbifrost import _bf, BFarray
from bifrost_b200.candidates import Candidates, RECORD_FIELDS
from bifrost_b200.blocks.candidates import candidate_header, candidate_lines
from bifrost_b200.blocks.pulse_search import pulse_search_header
from oracle import candidates as oc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

S = _bf


# ------------------------------------------------------------------ oracle (CPU)
def brute_force(peaks, threshold, tr, pr, decim):
    """Records straight from the definition: every pair tested, then BFS."""
    p = np.asarray(peaks, np.float32)
    ntrial, nblk, nfield = p.shape
    mem = []
    for j in range(nblk):
        for t in range(ntrial):
            s, o = float(p[t, j, 0]), float(p[t, j, 1])
            if s >= threshold and 0 <= o < decim:
                mem.append((j * ntrial + t, t, j, float(j * decim) + o))
    n = len(mem)
    adj = [[b for b in range(n) if b != a and abs(mem[a][1] - mem[b][1]) <= tr
            and abs(mem[a][3] - mem[b][3]) <= pr] for a in range(n)]
    seen, out = [False] * n, []
    for a in range(n):                     # members are in k order: each cluster starts at its smallest k
        if seen[a]:
            continue
        comp, q = [], deque([a])
        seen[a] = True
        while q:
            x = q.popleft()
            comp.append(x)
            for y in adj[x]:
                if not seen[y]:
                    seen[y] = True
                    q.append(y)
        rep = min(comp, key=lambda x: (-float(p[mem[x][1], mem[x][2], 0]), mem[x][0]))
        k, t, j, pos = mem[rep]
        ts, ps = [mem[x][1] for x in comp], [mem[x][3] for x in comp]
        out.append([float(p[t, j, 0]), t, pos, float(p[t, j, 2]) if nfield == 3 else 0., len(comp),
                    min(ts), max(ts), min(ps), max(ps)])
    return np.array(out, np.float64).reshape(-1, 9)


def random_map(rng, ntrial, nblk, decim, nfield=3, density=0.2, frac=False):
    p = np.empty((ntrial, nblk, nfield), np.float32)
    p[..., 0] = np.where(rng.random((ntrial, nblk)) < density, rng.uniform(5, 9, (ntrial, nblk)),
                         rng.uniform(-2, 4.9, (ntrial, nblk)))
    off = rng.integers(0, decim, (ntrial, nblk)).astype(np.float32)
    if frac:
        off += rng.random((ntrial, nblk)).astype(np.float32) * 0.999
        off = np.minimum(off, np.float32(decim) - np.float32(decim) * np.float32(2 ** -23))
    p[..., 1] = off
    if nfield > 2:
        p[..., 2:] = rng.integers(1, 64, (ntrial, nblk, nfield - 2))
    return p


@pytest.mark.parametrize('seed', range(8))
def test_oracle_equals_brute_force(seed):
    rng = np.random.default_rng(seed)
    ntrial, nblk = int(rng.integers(1, 14)), int(rng.integers(1, 30))
    decim = int(rng.choice([1, 3, 7, 16]))
    tr, pr = int(rng.integers(0, 4)), int(rng.integers(0, 3 * decim + 2))
    p = random_map(rng, ntrial, nblk, decim, nfield=2 + seed % 2, density=0.3, frac=seed % 3 == 0)
    p[..., 0] = np.round(p[..., 0] * 2) / 2          # equal scores happen
    got = oc.cluster(p, 6.0, tr, pr, decim)
    want = brute_force(p, 6.0, tr, pr, decim)
    assert got.shape == want.shape
    assert np.array_equal(got, want)


def one_row_map(ntrial, nblk, cells, nfield=3):
    """All-below-threshold map with members {(t, j): (score, offset)}."""
    p = np.zeros((ntrial, nblk, nfield), np.float32)
    for (t, j), (s, o) in cells.items():
        p[t, j, 0], p[t, j, 1] = s, o
        if nfield == 3:
            p[t, j, 2] = 4
    return p


def test_oracle_radius_edges():
    decim = 10
    # pos 3 and 3 + R_p link; 3 + R_p + 1 does not
    for pr, link in ((7, True), (6, False)):
        p = one_row_map(1, 3, {(0, 0): (7., 3.), (0, 1): (8., 0.)})
        r = oc.cluster(p, 6., 0, pr, decim)
        assert len(r) == (1 if link else 2)
    # |dt| = R_t links, R_t + 1 does not
    for tr, link in ((3, True), (2, False)):
        p = one_row_map(5, 1, {(0, 0): (7., 1.), (3, 0): (8., 1.)})
        assert len(oc.cluster(p, 6., tr, 0, decim)) == (1 if link else 2)


def test_oracle_links_across_block_boundary():
    p = one_row_map(2, 4, {(0, 1): (7., 9.), (1, 2): (8., 0.)})
    r = oc.cluster(p, 6., 1, 1, 10)
    assert len(r) == 1
    assert list(r[0]) == [8., 1., 20., 4., 2., 0., 1., 19., 20.]


def test_oracle_equal_scores_pick_smaller_k():
    # k = j ntrial + t: (2, 0) has k 2, (0, 1) has k 3
    p = one_row_map(3, 2, {(0, 1): (7., 0.), (2, 0): (7., 5.), (1, 0): (6.5, 9.)})
    r = oc.cluster(p, 6., 2, 10, 10)
    assert len(r) == 1 and r[0, 1] == 2 and r[0, 2] == 5.
    p[..., 0] = -5.                                      # -0 and +0 tie too
    p[2, 0, 0] = -0.
    p[0, 1, 0] = 0.
    r = oc.cluster(p, -0.5, 2, 10, 10)
    assert len(r) == 1 and r[0, 1] == 2 and np.signbit(r[0, 0])


def test_oracle_nan_and_offset_range():
    cells = {(0, 0): (np.nan, 1.), (1, 0): (7., np.nan), (2, 0): (7., -1.), (3, 0): (7., 10.),
             (4, 0): (7., -0.), (5, 0): (7., 9.5), (6, 0): (np.inf, 2.)}
    p = one_row_map(7, 1, cells)
    r = oc.cluster(p, 6., 0, 0, 10)
    assert [int(x) for x in r[:, 1]] == [4, 5, 6]
    assert r[0, 2] == 0. and not np.signbit(r[0, 2]) and r[1, 2] == 9.5 and r[2, 0] == np.inf


def test_oracle_threshold_equality():
    p = one_row_map(2, 1, {(0, 0): (6., 0.), (1, 0): (np.nextafter(np.float32(6.), np.float32(0)), 0.)})
    r = oc.cluster(p, 6., 0, 0, 1)
    assert len(r) == 1 and r[0, 1] == 0
    assert len(oc.cluster(p, 6.000000000001, 0, 0, 1)) == 0   # the compare is fp64


# ------------------------------------------------------------------ headers and lines (CPU)
def peak_header(ndm=120, decim=256, widths=(1, 2, 4, 8, 16, 32), labels=None):
    bank = {'_tensor': {'dtype': 'f32', 'shape': [ndm, -1], 'labels': ['dispersion', 'time'],
                        'scales': [[1.5, 0.25], [100., 1e-3]], 'units': ['pc cm^-3', 's']},
            'name': 'obs/fil', 'gulp_nframe': 4096}
    h = pulse_search_header(bank, widths, decim)
    if labels is not None:
        h['_tensor']['labels'] = labels
    return h


def test_pulse_search_header_peak_decim():
    h = peak_header(decim=128)
    assert h['peak_decim'] == 128
    assert h['_tensor']['scales'][1] == [100., 1e-3 * 128]


def test_candidate_header():
    decim, tsamp, dm0, ddm, widest = candidate_header(peak_header(decim=128, widths=(1, 3, 17)))
    assert (decim, dm0, ddm, widest) == (128, 1.5, 0.25, 17)
    assert abs(tsamp - 1e-3) < 1e-18
    with pytest.raises(KeyError):
        candidate_header(peak_header(labels=['freq', 'time', 'peak']))
    h = peak_header()
    t = h['_tensor']
    beams = deepcopy(h)
    for key, v in (('shape', 2), ('labels', 'beam'), ('scales', None), ('units', None)):
        beams['_tensor'][key].insert(0, v)
    with pytest.raises(KeyError):
        candidate_header(beams)
    with pytest.raises(KeyError):
        candidate_header({k: v for k, v in h.items() if k != 'peak_decim'})
    with pytest.raises(TypeError):
        candidate_header(dict(h, _tensor=dict(t, dtype='f64')))


def test_candidate_lines():
    rec = np.array([[12.5, 7, 300., 16, 42, 5, 9, 290., 311.],
                    [6.25, 0, 0., 1, 1, 0, 0, 0., 0.]])
    lines = candidate_lines(rec, 4096, 1e-3, 1.5, 0.25)
    assert lines == ['12.500000\t4396\t4.396000000\t16\t7\t3.250000\t42\t4386\t4407\n',
                     '6.250000\t4096\t4.096000000\t1\t0\t1.500000\t1\t4096\t4096\n']
    assert candidate_lines(np.zeros((0, 9)), 0, 1e-3, 0., 1.) == []
    assert RECORD_FIELDS == ['snr', 'trial', 'pos', 'width', 'members', 'trial_lo', 'trial_hi', 'pos_lo',
                             'pos_hi']


@pytest.mark.parametrize('args', [(float('nan'), 8, 32, 16), (float('inf'), 8, 32, 16), (6., -1, 32, 16),
                                  (6., 33, 32, 16), (6., 8, -1, 16), (6., 8, 32 * 16 + 1, 16),
                                  (6., 8, 32, 0), (6., 8, 32, (1 << 24) + 1)])
def test_init_rejects_bad_arguments(args):
    with pytest.raises(RuntimeError, match='INVALID_ARGUMENT'):
        Candidates().init(*args)


def test_init_accepts_limits():
    Candidates().init(-1e30, 32, 32 * 16, 16)
    Candidates().init(6., 0, 0, 1 << 24)


# ------------------------------------------------------------------ descriptor-only statuses (CPU)
DUMMY = 1 << 32            # 4096-aligned, never dereferenced
NBYTE = {'f32': 4, 'f64': 8, 'i32': 4, 'i64': 8}
DTYPE = {'f32': S.BF_DTYPE_F32, 'f64': S.BF_DTYPE_F64, 'i32': S.BF_DTYPE_I32, 'i64': S.BF_DTYPE_I64}


def desc(dtype, shape, last_stride=None):
    a = BFarray()
    a.data = DUMMY
    a.space = S.BF_SPACE_CUDA
    a.dtype = DTYPE[dtype]
    a.ndim = len(shape)
    stride = last_stride or NBYTE[dtype]
    for d in reversed(range(len(shape))):
        a.shape[d] = shape[d]
        a.strides[d] = stride
        stride *= shape[d]
    return a


def exec_desc(plan, peaks, table, count, ptr, size):
    return S.bfCandidatesExecute(plan, ctypes.byref(peaks), ctypes.byref(table), ctypes.byref(count), ptr, size)


@pytest.fixture
def plan():
    p = ctypes.c_void_p()
    assert S.bfCandidatesCreate(ctypes.byref(p)) == S.BF_STATUS_SUCCESS
    yield p
    assert S.bfCandidatesDestroy(p) == S.BF_STATUS_SUCCESS


# (leading dims, ntrial, nblk, nfield, ncap, workspace bytes of the (NULL, &size) query)
QUERY = [((2, 5), 100, 3, 3, 16, 24064 + 12032 + 256 + 6400),
         ((), 794, 512, 3, 4096, 3252224 + 1626112 + 1024 + 163840),
         ((3,), 1, 1, 2, 0, 256 * 3)]


@pytest.mark.parametrize('lead,ntrial,nblk,nfield,ncap,size', QUERY)
def test_query_size_and_storage_refusals(plan, lead, ntrial, nblk, nfield, ncap, size):
    lead = list(lead)
    assert S.bfCandidatesInit(plan, 6., 8, 32, 16) == S.BF_STATUS_SUCCESS
    arrays = (desc('f32', lead + [ntrial, nblk, nfield]), desc('f64', lead + [ncap, 9]), desc('i32', lead + [1]))
    got = S.BFsize(0)
    assert exec_desc(plan, *arrays, None, ctypes.byref(got)) == S.BF_STATUS_SUCCESS
    assert got.value == size
    short = S.BFsize(size - 1)
    assert exec_desc(plan, *arrays, DUMMY, ctypes.byref(short)) == S.BF_STATUS_INSUFFICIENT_STORAGE
    assert exec_desc(plan, *arrays, DUMMY, None) == S.BF_STATUS_INVALID_ARGUMENT


def test_descriptor_statuses(plan):
    size = S.BFsize(0)
    good = (desc('f32', [2, 50, 10, 3]), desc('f64', [2, 8, 9]), desc('i32', [2, 1]))

    def st(*arrays):
        return exec_desc(plan, *arrays, None, ctypes.byref(size))

    assert st(*good) == S.BF_STATUS_INVALID_STATE                  # not initialised
    assert S.bfCandidatesInit(plan, 6., 8, 32, 16) == S.BF_STATUS_SUCCESS
    assert st(*good) == S.BF_STATUS_SUCCESS
    p, t, c = good
    assert st(desc('f64', [2, 50, 10, 3]), t, c) == S.BF_STATUS_UNSUPPORTED_DTYPE
    assert st(p, desc('f32', [2, 8, 9]), c) == S.BF_STATUS_UNSUPPORTED_DTYPE
    assert st(p, t, desc('i64', [2, 1])) == S.BF_STATUS_UNSUPPORTED_DTYPE
    for bad in (desc('f32', [2, 50, 10, 4]), desc('f32', [2, 50, 10, 1]), desc('f32', [3, 50, 10, 3]),
                desc('f32', [50, 10, 3])):
        assert st(bad, t, c) == S.BF_STATUS_INVALID_SHAPE
    for bad in (desc('f64', [2, 8, 8]), desc('f64', [3, 8, 9]), desc('f64', [8, 9])):
        assert st(p, bad, c) == S.BF_STATUS_INVALID_SHAPE
    for bad in (desc('i32', [2, 2]), desc('i32', [3, 1]), desc('i32', [2])):
        assert st(p, t, bad) == S.BF_STATUS_INVALID_SHAPE
    assert st(desc('f32', [2, 50, 10, 3], last_stride=8), t, c) == S.BF_STATUS_UNSUPPORTED_STRIDE
    assert st(p, desc('f64', [2, 8, 9], last_stride=16), c) == S.BF_STATUS_UNSUPPORTED_STRIDE
    odd = desc('f32', [2, 50, 10, 3])
    odd.strides[1] = 122                                             # trial stride not whole elements
    assert st(odd, t, c) == S.BF_STATUS_UNSUPPORTED_STRIDE
    big = desc('f32', [1 << 16, 1 << 15, 3])                         # ntrial nblk = 2^31
    assert st(big, desc('f64', [8, 9]), desc('i32', [1])) == S.BF_STATUS_UNSUPPORTED_SHAPE
    assert S.bfCandidatesInit(plan, 6., 8, 16, 1 << 24) == S.BF_STATUS_SUCCESS
    wide = desc('f32', [1, 128, 3])                                  # nblk decim = 2^31
    assert st(wide, desc('f64', [8, 9]), desc('i32', [1])) == S.BF_STATUS_UNSUPPORTED_SHAPE


def test_handle_statuses():
    size = S.BFsize(0)
    arrays = (desc('f32', [5, 10, 3]), desc('f64', [4, 9]), desc('i32', [1]))
    assert S.bfCandidatesCreate(None) == S.BF_STATUS_INVALID_POINTER
    assert S.bfCandidatesDestroy(None) == S.BF_STATUS_INVALID_HANDLE
    assert exec_desc(None, *arrays, None, ctypes.byref(size)) == S.BF_STATUS_INVALID_HANDLE
    assert S.bfCandidatesInit(None, 6., 8, 32, 16) == S.BF_STATUS_INVALID_HANDLE
    p = ctypes.c_void_p()
    assert S.bfCandidatesCreate(ctypes.byref(p)) == S.BF_STATUS_SUCCESS
    assert exec_desc(p, *arrays, None, ctypes.byref(size)) == S.BF_STATUS_INVALID_STATE
    assert S.bfCandidatesExecute(p, None, None, None, None, ctypes.byref(size)) == S.BF_STATUS_INVALID_POINTER
    assert S.bfCandidatesDestroy(p) == S.BF_STATUS_SUCCESS


# ------------------------------------------------------------------ GPU
SENTINEL = -123.25


def run(peaks, threshold, tr, pr, decim, ncap, d_peaks=None, plan=None):
    """GPU table and count for a host map [..., ntrial, nblk, nfield] (or the
    device view d_peaks of it), the table pre-filled with SENTINEL."""
    p = np.asarray(peaks)
    lead = p.shape[:-3]
    d_p = d_peaks if d_peaks is not None else bf.asarray(np.ascontiguousarray(p), space='cuda')
    d_t = bf.asarray(np.full(lead + (ncap, 9), SENTINEL), space='cuda')
    d_c = bf.asarray(np.full(lead + (1,), -7, np.int32), space='cuda')
    if plan is None:
        plan = Candidates()
        plan.init(threshold, tr, pr, decim)
    plan.execute(d_p, d_t, d_c)
    bf.device.stream_synchronize()
    return np.asarray(d_t.copy('system')), np.asarray(d_c.copy('system'))


def check(table, count, peaks, threshold, tr, pr, decim):
    """Bit for bit against the oracle; rows past min(count, ncap) untouched."""
    recs, want_count = oc.candidates(peaks, threshold, tr, pr, decim)
    assert np.array_equal(count, want_count)
    lead = table.shape[:-2]
    ncap = table.shape[-2]
    for i, idx in enumerate(np.ndindex(*lead)):
        n = min(len(recs[i]), ncap)
        assert np.array_equal(table[idx][:n].view(np.uint64), recs[i][:n].view(np.uint64)), idx
        assert np.all(table[idx][n:] == SENTINEL)
    return recs


RANDOM = {   # name: (lead, ntrial, nblk, nfield, decim, tr, pr, density, frac)
    'basic':     ((), 60, 200, 3, 16, 4, 24, 0.05, False),
    'batch':     ((2, 3), 40, 90, 3, 7, 2, 10, 0.1, False),
    'ntrial1':   ((), 1, 3000, 3, 5, 8, 9, 0.2, False),
    'nblk1':     ((4,), 500, 1, 2, 33, 3, 33, 0.3, False),
    'odd_decim': ((), 97, 301, 3, 13, 32, 13 * 32, 0.02, False),
    'frac':      ((), 50, 120, 2, 3, 1, 4, 0.15, True),
    'decim1':    ((), 30, 700, 3, 1, 5, 32, 0.1, False),
    'pr0':       ((), 64, 64, 3, 8, 0, 0, 0.5, False),
}


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(RANDOM))
@pytest.mark.parametrize('seed', [0, 1, 2])
def test_matches_oracle(name, seed):
    lead, ntrial, nblk, nfield, decim, tr, pr, density, frac = RANDOM[name]
    rng = np.random.default_rng(1000 * seed + sorted(RANDOM).index(name))
    p = np.stack([random_map(rng, ntrial, nblk, decim, nfield, density, frac)
                  for _ in range(int(np.prod(lead, dtype=int)))]).reshape(lead + (ntrial, nblk, nfield))
    p[..., 0] = np.round(p[..., 0] * 4) / 4
    table, count = run(p, 6., tr, pr, decim, 4096)
    recs = check(table, count, p, 6., tr, pr, decim)
    assert sum(len(r) for r in recs) > 0


@pytest.mark.gpu
def test_diagonal_chain_is_one_cluster():
    ntrial, nblk, decim = 200, 5000, 10
    p = np.zeros((ntrial, nblk, 3), np.float32)
    j = np.arange(nblk)
    t = np.abs((j % (2 * ntrial - 2)) - (ntrial - 1))    # sweeps the trials up and down
    p[t, j, 0] = 7. + (j % 13) / 8
    p[t, j, 1] = 9 - (j % 10)                             # consecutive members 1..19 samples apart
    table, count = run(p, 6., 1, 19, decim, 8)
    assert count[0] == 1
    check(table, count, p, 6., 1, 19, decim)
    assert table[0, 4] == nblk and table[0, 5] == 0 and table[0, 6] == ntrial - 1


@pytest.mark.gpu
def test_lattice_forms_no_links():
    tr, pr, decim = 3, 20, 8
    ntrial, nblk = 64, 400
    p = np.zeros((ntrial, nblk, 3), np.float32)
    pos = np.arange(0, nblk * decim, pr + 1)
    for t in range(0, ntrial, tr + 1):
        p[t, pos // decim, 0] = 8.
        p[t, pos // decim, 1] = pos % decim
    table, count = run(p, 6., tr, pr, decim, 4096)
    assert count[0] == len(pos) * len(range(0, ntrial, tr + 1))
    check(table, count, p, 6., tr, pr, decim)
    assert np.all(table[:count[0], 4] == 1)


@pytest.mark.gpu
def test_dense_map_is_one_cluster():
    rng = np.random.default_rng(3)
    p = random_map(rng, 300, 800, 16, 3, density=0.)
    table, count = run(p, -10., 1, 32, 16, 4)
    assert count[0] == 1 and table[0, 4] == 300 * 800
    check(table, count, p, -10., 1, 32, 16)


@pytest.mark.gpu
def test_overflow_keeps_first_clusters():
    tr, pr, decim = 1, 4, 4
    p = np.zeros((40, 300, 3), np.float32)
    p[::2, ::2, 0] = np.arange(20 * 150).reshape(20, 150) % 7 + 6
    table, count = run(p, 6., tr, pr, decim, 5)
    assert count[0] == 20 * 150
    check(table, count, p, 6., tr, pr, decim)


@pytest.mark.gpu
def test_strided_leading_dims():
    rng = np.random.default_rng(4)
    # [2, 3] batch with padded trial rows and a peak axis of 4 (the first 3 used)
    big = np.stack([random_map(rng, 30, 50, 4, 4, 0.1) for _ in range(6)]).reshape(2, 3, 30, 50, 4)
    big[..., 0] = np.round(big[..., 0] * 4) / 4
    d_big = bf.asarray(big, space='cuda')
    view = d_big.transpose((1, 0, 2, 3, 4))[:, :, 1:, :, :3]          # [3, 2, 29, 50, 3]
    host = np.ascontiguousarray(big.transpose(1, 0, 2, 3, 4)[:, :, 1:, :, :3])
    table, count = run(host, 6., 2, 6, 4, 64, d_peaks=view)
    check(table, count, host, 6., 2, 6, 4)
    # a period_search map [ndm, time, harmonic, nblk, 2] searched as [time, harmonic, ndm, nblk, 2]
    ps = np.stack([random_map(rng, 1, 70, 16, 2, 0.1)[0] for _ in range(40 * 3 * 2)]).reshape(40, 3, 2, 70, 2)
    d_ps = bf.asarray(ps, space='cuda')
    pview = d_ps.transpose((1, 2, 0, 3, 4))
    phost = np.ascontiguousarray(ps.transpose(1, 2, 0, 3, 4))
    table, count = run(phost, 6., 4, 40, 16, 128, d_peaks=pview)
    check(table, count, phost, 6., 4, 40, 16)


def config2_map(decim, seed):
    """A [794, 131072 / decim, 3] map: N(0, 1.3) scores with a few bright
    smeared blobs, integer offsets, power-of-two widths."""
    rng = np.random.default_rng(seed)
    nblk = 131072 // decim
    p = np.empty((794, nblk, 3), np.float32)
    p[..., 0] = rng.normal(0, 1.3, (794, nblk))
    for r, j in ((150, nblk // 7), (397, nblk // 2), (700, (4 * nblk) // 5)):
        p[max(0, r - 30):r + 30, j:j + 3, 0] += 12.
    p[..., 1] = rng.integers(0, decim, (794, nblk))
    p[..., 2] = 2 ** rng.integers(0, 9, (794, nblk))
    return p


@pytest.mark.gpu
@pytest.mark.parametrize('decim,threshold', [(256, 6.), (16, 5.)])
def test_config2_repeatability(decim, threshold):
    p = config2_map(decim, 5)
    d_p = bf.asarray(p, space='cuda')
    plan = Candidates()
    plan.init(threshold, 8, 256, decim)
    a, ca = run(p, threshold, 8, 256, decim, 4096, d_peaks=d_p, plan=plan)
    b, cb = run(p, threshold, 8, 256, decim, 4096, d_peaks=d_p, plan=plan)
    assert np.array_equal(ca, cb) and np.array_equal(a.view(np.uint64), b.view(np.uint64))
    check(a, ca, p, threshold, 8, 256, decim)
    assert ca[0] >= 3


@pytest.mark.gpu
def test_workspace_modes():
    rng = np.random.default_rng(6)
    p = np.stack([random_map(rng, 50, 300, 8, 3, 0.05) for _ in range(3)])
    d_p = bf.asarray(p, space='cuda')
    plan = Candidates()
    plan.init(6., 3, 12, 8)
    tabs = [bf.asarray(np.full((3, 100, 9), SENTINEL), space='cuda') for _ in range(2)]
    cnts = [bf.zeros((3, 1), 'i32', 'cuda') for _ in range(2)]
    size = plan.get_workspace_size(d_p, tabs[0], cnts[0])             # (NULL, &size): query only
    assert size > 0
    bf.device.stream_synchronize()
    assert np.all(np.asarray(tabs[0].copy('system')) == SENTINEL)
    assert np.all(np.asarray(cnts[0].copy('system')) == 0)
    plan.execute(d_p, tabs[0], cnts[0])                                # (NULL, NULL): library-managed
    ws = bf.empty((size,), dtype='u8', space='cuda')
    plan.execute_workspace(d_p, tabs[1], cnts[1], ws.ctypes.data, size)  # (ptr, &size): caller's memory
    bf.device.stream_synchronize()
    a, b = (np.asarray(x.copy('system')) for x in tabs)
    ca, cb = (np.asarray(x.copy('system')) for x in cnts)
    assert np.array_equal(ca, cb) and np.array_equal(a.view(np.uint64), b.view(np.uint64))
    check(a, ca, p, 6., 3, 12, 8)
    short = S.BFsize(size - 1)
    assert S.bfCandidatesExecute(plan.obj, d_p.as_BFarray(), tabs[1].as_BFarray(), cnts[1].as_BFarray(),
                                 ctypes.c_void_p(ws.ctypes.data), ctypes.byref(short)) == \
        S.BF_STATUS_INSUFFICIENT_STORAGE


@pytest.mark.gpu
def test_fixed_kernel_list():
    from kernel_trace import device_kernels
    rng = np.random.default_rng(7)
    sparse = random_map(rng, 200, 500, 16, 3, 0.001)
    dense = random_map(rng, 200, 500, 16, 3, 1.)
    plan = Candidates()
    plan.init(6., 8, 32, 16)
    d_t = bf.zeros((64, 9), 'f64', 'cuda')
    d_c = bf.zeros((1,), 'i32', 'cuda')
    lists = []
    for p in (sparse, dense):
        d_p = bf.asarray(p, space='cuda')
        plan.execute(d_p, d_t, d_c)                                    # workspace allocated outside the trace
        lists.append(device_kernels(lambda: plan.execute(d_p, d_t, d_c)))
    assert lists[0] == lists[1]
    assert len(lists[0]) == 7
    for name, stage in zip(lists[0], ('mark', 'link', 'flatten', 'scan', 'assign', 'reduce', 'write')):
        assert 'candidates_%s_kernel' % stage in name


# ------------------------------------------------------------------ pipeline
@pytest.mark.gpu
def test_fdmt_pulse_search_candidates_pipeline(tmp_path):
    from bifrost_b200 import blocks
    from bifrost_b200.pipeline import Pipeline
    from test_pulse_search import filterbank
    nchan, md, gulp, ntime = 256, 120, 4096, 3 * 4096 + 600
    f0, df, dt = 1200., 0.5, 1e-3
    widths, decim, threshold, tr = (1, 2, 4, 8, 16, 32), 256, 6.0, 8
    pulses = ((0.2, 2000), (0.5, 4090), (0.9, 9000))          # the second straddles a gulp boundary
    x, rows = filterbank(nchan, ntime, md, f0, df, pulses, 11)
    hdr = {'_tensor': {'dtype': 'i8', 'shape': [-1, nchan], 'labels': ['time', 'freq'],
                       'scales': [[0, dt], [f0, df]], 'units': ['s', 'MHz']},
           'name': 'fil', 'gulp_nframe': gulp}
    peaks, heads = [], []
    with Pipeline() as p:
        src = blocks.array_source(x, hdr, gulp_nframe=gulp)
        b = blocks.copy(src, space='cuda')
        b = blocks.transpose(b, ['freq', 'time'])
        d = blocks.fdmt(b, max_delay=md)
        s = blocks.pulse_search(d, widths=widths, decim=decim)
        blocks.callback_sink(blocks.copy(s, space='system'), lambda q: heads.append(deepcopy(q.header)),
                             lambda q: peaks.append(np.array(q.data)))
        blocks.write_candidates(s, path=str(tmp_path), threshold=threshold, trial_radius=tr)
        p.run()
    got = np.concatenate(peaks, axis=1)
    text = (tmp_path / 'fil.cand').read_text()
    # the file is the oracle applied gulp by gulp, at the widest boxcar as pos_radius
    _, tsamp, dm0, ddm, widest = candidate_header(heads[0])
    assert widest == 32 and abs(tsamp - dt) < 1e-15
    per = gulp // decim
    want, spans = [], []
    for f in range(0, got.shape[1], per):
        recs = oc.cluster(got[:, f:f + per], threshold, tr, widest, decim)
        want += candidate_lines(recs, f * decim, tsamp, dm0, ddm)
        spans.append((f * decim, recs))
    assert text == ''.join(want)
    cands = np.array([[float(v) for v in line.split('\t')] for line in text.splitlines()])
    # each injected pulse is the brightest candidate of its gulp within 1024 samples, at its DM and time
    for (frac, t0), row in zip(pulses, rows):
        g0 = (t0 // gulp) * gulp
        near = cands[(np.abs(cands[:, 1] - t0) <= 1024) & (cands[:, 1] >= g0) & (cands[:, 1] < g0 + gulp)]
        best = near[np.argmax(near[:, 0])]
        assert abs(best[4] - row) <= 2, (best, row)
        assert abs(best[1] - t0) <= best[3] + 1, (best, t0)
        if t0 % gulp < gulp - 64:
            assert len(near) == 1, near
    # the straddling pulse: its cells in the next gulp form a candidate of their own there
    after = cands[(cands[:, 7] >= gulp) & (cands[:, 7] < gulp + 64)]
    assert len(after) >= 1
    assert np.all((cands[:, 7] >= gulp) | (cands[:, 8] < gulp))       # no candidate spans the boundary
