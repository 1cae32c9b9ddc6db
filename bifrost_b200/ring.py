"""Ring buffers between blocks, in the memory space of the data they carry.

The reference's ring (src/ring_impl.cpp, python/bifrost/ring2.py) is a
byte-addressed circular buffer with a *ghost region*: the first `ghost` bytes
are mirrored behind the end of the buffer so that every span a reader or
writer asks for is contiguous, and the mirror is maintained when spans are
committed (ring_impl.cpp:273-288: `_ghost_write` / `_ghost_read`).  This is the
same machine, frame-addressed, for the blocks of the hot path:

  * one allocation per sequence, in the ring's space -- 'cuda' rings live in
    device memory and their ghost copies are device-to-device copies issued
    on the committing thread's stream (bfArrayCopy), never staged on the host;
  * the tensor's frame axis is the circular axis; axes in front of it are
    the reference's "ringlets" (ring2.py:87-107): a span is then a strided
    view, which is what the kernels take (DESIGN.md section 3);
  * one writer, any number of readers, each with its own cursor; the writer
    blocks when it would overwrite frames a *guaranteed* reader has not
    released, a reader blocks until the frames it wants are committed or the
    sequence ends (ring_impl.cpp:open_read_at / reserve_span).  A reader opened
    with guarantee=False never holds the writer back: a span any frame of
    which has been overwritten comes back empty with `nframe_skipped` set, and
    `Reader.overwritten()` tells after the fact whether the writer got there
    while the span was in use (ring.h:bfRingSpanGetSizeOverwritten);
  * storage is sized when the sequence starts, from the spans the writer and
    every reader declare (gulp + overlap), `buffer_nframe` / `buffer_factor`
    of the block scope (pipeline.py:84-134 of the reference).

Everything here is host-side bookkeeping (a mutex and a condition variable per
ring); the data path is the copies at the seam.
"""
import threading
from copy import deepcopy

import numpy as np

from bifrost_b200 import device
from bifrost_b200.DataType import DataType
from bifrost_b200.ndarray import ndarray, empty, copy_array


class PipelineAborted(Exception):
    """Raised inside blocked ring calls when another block failed."""


class EndOfData(Exception):
    pass


def frame_axis(tensor):
    return tensor['shape'].index(-1)


def _frame_nbit(tensor):
    n = DataType(tensor['dtype']).itemsize_bits
    for s in tensor['shape']:
        if s != -1:
            n *= s
    return n


def slice_frames(arr, axis, lo, hi):
    sl = [slice(None)] * arr.ndim
    sl[axis] = slice(lo, hi)
    return arr[tuple(sl)]


class Sequence(object):
    """One sequence as readers see it: header + tensor description."""

    def __init__(self, header, index=0):
        self.header = header
        self.tensor = header['_tensor']
        self.name = header.get('name', '')
        self.time_tag = header.get('time_tag', 0)
        self.index = index


class Span(object):
    def __init__(self, sequence, data, frame_offset, faxis):
        self.sequence = sequence
        self.tensor = sequence.tensor
        self.data = data
        self.frame_offset = frame_offset
        self.frame_axis = faxis
        self.nframe = data.shape[faxis]
        self.nframe_skipped = 0
        self._lost_query = None     # set for spans of unguaranteed readers
        self.frame_nbyte = 0 if self.nframe == 0 else data.nbytes // max(self.nframe, 1)


def _nframe_overwritten(span):
    """Frames of the span the writer has taken back since it was acquired (all of
    them or none; always 0 for guaranteed readers) -- asked when read, like
    ring2.py:ReadSpan.nframe_overwritten of the reference."""
    return span.nframe if (span._lost_query is not None and span._lost_query()) else 0


Span.nframe_overwritten = property(_nframe_overwritten)


class _SeqState(object):
    """Writer-side state of one sequence (shared with the readers under the ring lock)."""

    def __init__(self, header, index, writer_span):
        self.seq = Sequence(header, index)
        self.faxis = frame_axis(self.seq.tensor)
        self.writer_span = max(1, int(writer_span))
        self.storage = None         # bf.ndarray [.., cap + ghost, ..]
        self.cap = 0
        self.ghost = 0
        self.head = 0               # frames committed
        self.reserved = 0           # frames of the open write span (the writer may scribble on them)
        self.ended = False
        self.opened = {}            # reader -> (gulp, overlap) once it has seen the header
        self.tails = {}             # reader -> frames released
        self.closed = set()


class Ring(object):
    def __init__(self, space, owner=None, name=None):
        self.space = str(space)
        self.owner = owner
        self.consumers = []         # blocks (graph bookkeeping; readers are opened by Pipeline.run)
        self.views = []
        self.name = name or f"ring_{id(self):x}"
        self.header_transform = None
        self.base = None
        self._lock = threading.Lock()
        self._cond = threading.Condition(self._lock)
        self._readers = []
        self._seqs = []             # _SeqState, in order
        self._writing = True
        self._abort = None
        self.buffer_nframe = None
        self.buffer_factor = None
        self.stats = dict(ghost_copies=0, ghost_frames=0, allocations=0)

    # ------------------------------------------------------------- plumbing
    def _check_abort(self):
        if self._abort is not None and self._abort.is_set():
            raise PipelineAborted()

    def _wait(self):
        self._cond.wait(0.2)
        self._check_abort()

    def set_abort_event(self, ev):
        self._abort = ev

    def wake(self):
        with self._cond:
            self._cond.notify_all()

    def root(self):
        return self

    def transform_header(self, hdr):
        return hdr

    def reinterpret(self, seq, data):
        return data

    # --------------------------------------------------------------- writer
    def begin_sequence(self, header, gulp_nframe):
        """Publishes a new sequence.  Storage is allocated by the first
        reserve(), once every reader has declared its span."""
        with self._cond:
            # readers must be done with the previous sequence before its storage goes away
            while self._seqs and any(r.guarantee and r not in self._seqs[-1].closed for r in self._readers):
                self._wait()
            if self._seqs:
                self._seqs[-1].storage = None
            st = _SeqState(deepcopy(header), len(self._seqs), gulp_nframe)
            self._seqs.append(st)
            self._cond.notify_all()
            return st

    def _allocate(self, st):
        span = st.writer_span
        for gulp, ovl in st.opened.values():
            span = max(span, gulp + ovl)
        factor = self.buffer_factor or 4
        cap = max(int(self.buffer_nframe or 0), factor * span, 2 * span)
        shape = list(st.seq.tensor['shape'])
        shape[st.faxis] = cap + span
        st.storage = empty(shape, dtype=st.seq.tensor['dtype'], space=self.space)
        st.cap, st.ghost = cap, span
        self.stats['allocations'] += 1

    def reserve(self, st, nframe):
        """A writable span of `nframe` frames following the committed ones."""
        with self._cond:
            self._check_abort()                               # Pipeline.shutdown() stops writers that never wait
            while len(st.opened) < len(self._readers):       # every reader has seen the header
                self._wait()
            if st.storage is None:
                self._allocate(st)
            assert nframe <= st.ghost, "write span longer than declared"
            while True:
                held = [t for r, t in st.tails.items() if r.guarantee]
                if not held or st.head + nframe - st.cap <= min(held):
                    break
                self._wait()
            st.reserved = nframe
            b = st.head % st.cap
            return Span(st.seq, slice_frames(st.storage, st.faxis, b, b + nframe), st.head, st.faxis)

    def commit(self, st, nframe):
        """Makes the first `nframe` frames of the last reserved span visible:
        ghost maintenance (device copies on this thread's stream, behind the
        kernels that filled the span), ONE stream synchronisation -- the
        per-gulp synchronisation of the reference's block loop
        (pipeline.py:628) -- and only then the new head."""
        if nframe > 0:
            b, cap, g = st.head % st.cap, st.cap, st.ghost
            e = b + nframe
            if e > cap:        # the span ran into the ghost region: fold it back to the start
                self._ghost_copy(st, cap, e, 0)
            if b < g:          # the span covers mirrored frames: refresh the mirror
                self._ghost_copy(st, b, min(e, g), cap + b)
        if self.space != 'system':
            device.stream_synchronize()
        with self._cond:
            st.head += nframe
            st.reserved = 0
            self._cond.notify_all()

    def _ghost_copy(self, st, lo, hi, dst_lo):
        if hi <= lo:
            return
        copy_array(slice_frames(st.storage, st.faxis, dst_lo, dst_lo + hi - lo),
                   slice_frames(st.storage, st.faxis, lo, hi))
        self.stats['ghost_copies'] += 1
        self.stats['ghost_frames'] += hi - lo

    def end_sequence(self, st):
        with self._cond:
            st.ended = True
            self._cond.notify_all()

    def end_writing(self):
        with self._cond:
            self._writing = False
            self._cond.notify_all()

    # --------------------------------------------------------------- readers
    def open_reader(self, who=None, guarantee=None):
        if guarantee is None:
            guarantee = getattr(who, 'guarantee', True)
        r = Reader(self, who, bool(guarantee))
        with self._cond:
            self._readers.append(r)
        return r


class ViewRing(object):
    """``block_view``: the parent's storage and cursors, another header."""

    def __init__(self, parent, header_transform):
        self.parent = parent
        self.header_transform = header_transform
        self.space = parent.space
        self.owner = parent.owner
        self.consumers = []
        self.views = []
        self.name = f"view_{id(self):x}"

    def root(self):
        return self.parent.root()

    def transform_header(self, hdr):
        hdr = self.parent.transform_header(hdr)
        out = self.header_transform(deepcopy(hdr))
        if out is None:
            raise ValueError("Header transform returned None")
        return out

    def open_reader(self, who=None, guarantee=None):
        r = self.root().open_reader(who, guarantee)
        r.view = self
        return r

    def reinterpret(self, seq, data):
        """Present `data` (a span of the parent) with this view's tensor."""
        tensor = seq.tensor
        shape = list(tensor['shape'])
        fax = shape.index(-1)
        known = int(np.prod([s for s in shape if s != -1])) if len(shape) > 1 else 1
        dt = DataType(tensor['dtype'])
        shape[fax] = (data.nbytes * 8) // (known * dt.itemsize_bits)
        if list(data.shape) == shape and data.bf.dtype == dt:
            return data
        strides = None
        if not data.flags['C_CONTIGUOUS']:
            strides = _view_strides(data, shape) if data.bf.dtype == dt else None
            if strides is None:
                raise ValueError("Header views need C-contiguous spans")
        return ndarray(space=data.bf.space, buffer=data.ctypes.data, shape=shape, dtype=dt, strides=strides,
                       native=data.bf.native, conjugated=data.bf.conjugated)


def _view_strides(data, shape):
    """Strides that present the strided span `data` with `shape` without a copy
    (e.g. axes merged inside a ringlet, after a transpose that left the frame
    axis inside), or None if there are none.  Found by numpy's no-copy reshape
    of a probe with data's strides that never touches the memory."""
    probe = np.lib.stride_tricks.as_strided(np.zeros(1, np.dtype((np.void, data.itemsize))),
                                            shape=data.shape, strides=data.strides)
    try:
        return np.reshape(probe, shape, copy=False).strides
    except ValueError:
        return None


class Reader(object):
    """One consumer's cursor into a ring."""

    def __init__(self, ring, who=None, guarantee=True):
        self.ring = ring
        self.who = who
        self.guarantee = guarantee
        self.view = None
        self._next = 0
        self._num, self._den = 1, 1      # frames of the ring per frame of this reader's view

    def sequences(self):
        """Yields (state, Sequence-as-this-reader-sees-it) until the writer stops."""
        ring = self.ring
        while True:
            with ring._cond:
                while len(ring._seqs) <= self._next:
                    if not ring._writing:
                        return
                    ring._wait()
                st = ring._seqs[self._next]
            self._next += 1
            hdr = deepcopy(st.seq.header)
            self._num, self._den = 1, 1
            if self.view is not None:
                hdr = self.view.transform_header(hdr)
                # a view that splits or merges the frame axis (views.split_axis /
                # merge_axes) changes what a frame is: this reader counts in its
                # own frames, the ring in the writer's
                mine, theirs = _frame_nbit(hdr['_tensor']), _frame_nbit(st.seq.tensor)
                if mine != theirs:
                    if mine % theirs and theirs % mine:
                        raise ValueError("Header view changes the frame size by a non-integer factor")
                    self._num, self._den = (mine // theirs, 1) if mine > theirs else (1, theirs // mine)
            yield st, Sequence(hdr, st.seq.index)

    def _ring_frames(self, nframe, round_up=False):
        """This reader's frame count in frames of the ring."""
        n = nframe * self._num
        if n % self._den and not round_up:
            raise ValueError(f"{nframe} frames of the view are not a whole number of ring frames "
                             f"(1 ring frame = {self._den} view frames): choose gulp_nframe accordingly")
        return -(-n // self._den)

    def open(self, st, gulp, overlap):
        with self.ring._cond:
            st.opened[self] = (max(1, self._ring_frames(int(gulp), True)), max(0, self._ring_frames(int(overlap), True)))
            st.tails[self] = 0
            self.ring._cond.notify_all()

    def acquire(self, st, seq, frame_offset, nframe):
        """Frames [frame_offset, frame_offset + nframe) -- fewer at the end of the
        sequence, none (nframe 0) once it is exhausted."""
        ring = self.ring
        view_offset = frame_offset
        frame_offset, nframe = self._ring_frames(frame_offset), self._ring_frames(nframe)
        with ring._cond:
            while st.head < frame_offset + nframe and not st.ended:
                ring._wait()
            n = max(0, min(nframe, st.head - frame_offset))
            storage = st.storage            # (the writer drops it when the next sequence begins)
            if storage is None:
                n = 0
            if self._num > 1:
                n -= n % self._num                          # whole frames of the view only
            # an unguaranteed reader that was lapped: the span is void as a whole
            lost = (not self.guarantee) and n > 0 and frame_offset < st.head + st.reserved - st.cap
        if n == 0 or lost:
            shape = list(seq.tensor['shape'])
            shape[frame_axis(seq.tensor)] = 0
            span = Span(seq, empty(shape, dtype=seq.tensor['dtype'], space='system'), view_offset, frame_axis(seq.tensor))
            if lost:
                span.nframe_skipped = n * self._den // self._num
            return span
        b = frame_offset % st.cap
        data = slice_frames(storage, st.faxis, b, b + n)
        frame_offset = view_offset
        if not self.guarantee:
            span = Span(seq, self.view.reinterpret(seq, data) if self.view is not None else data,
                        frame_offset, frame_axis(seq.tensor))
            span._lost_query = lambda: self.overwritten(st, view_offset)
            return span
        if self.view is not None:
            data = self.view.reinterpret(seq, data)
        return Span(seq, data, frame_offset, frame_axis(seq.tensor))

    def overwritten(self, st, frame_offset):
        """True if the writer has (or may have) written over frames at or after
        `frame_offset` (this reader's frames) since they were acquired -- only an
        unguaranteed reader can see that happen."""
        if self.guarantee:
            return False
        first = frame_offset * self._num // self._den
        with self.ring._cond:
            return first < st.head + st.reserved - st.cap

    def release(self, st, upto_frame):
        upto_frame = upto_frame * self._num // self._den
        with self.ring._cond:
            st.tails[self] = max(st.tails.get(self, 0), upto_frame)
            self.ring._cond.notify_all()

    def close(self, st):
        with self.ring._cond:
            st.tails[self] = 1 << 62
            st.closed.add(self)
            self.ring._cond.notify_all()
