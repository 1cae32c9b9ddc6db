"""The block executor: the block API of the reference's ``bifrost.pipeline``
(python/bifrost/pipeline.py) -- ``SourceBlock`` / ``TransformBlock`` /
``SinkBlock`` with ``on_sequence`` / ``on_data``, ``block_view``,
``block_scope`` and ``Pipeline.run()`` -- on ring buffers that live in the
memory space of the data (bifrost_b200/ring.py).

As in the reference (pipeline.py:249-261, 558-650):
  * every block runs its own OS thread and its own CUDA stream (the library's
    per-thread stream), bound to the device named by ``gpu=`` and the core
    named by ``core=``;
  * blocks are connected by rings: the writer reserves a span, the block's
    ``on_data`` fills it, one stream synchronisation per gulp, commit; readers
    acquire spans of ``gulp + overlap`` frames and release them gulp by gulp;
  * a 'cuda' ring is device memory end to end -- a span handed to ``on_data``
    is a view of the ring, and wrapping is handled by device-side ghost copies;
  * headers are dicts with a ``_tensor`` entry (ring2.py:229-255), spans expose
    ``.data`` / ``.nframe`` / ``.frame_offset`` / ``.tensor``;
  * ``define_input_overlap_nframe`` re-presents the tail of each gulp to the
    next one (blocks/fdmt.py:112-115); ``on_data`` may return the number of
    frames to commit (blocks/accumulate.py:63-74).
An exception in any block stops the pipeline and is re-raised by ``run()``;
``shutdown()`` / ``shutdown_on_signals()`` stop it from outside.

``guarantee=False`` on a block (pipeline.py:518-537,590-643 of the reference)
makes its reader one the writer may lap: a gulp any frame of which was
overwritten -- before it was acquired or while ``on_data`` worked on it -- is
dropped as a whole, ``on_skip`` fills the corresponding output frames (zeros
by default) so the output keeps its cadence, and one more gulp is dropped
after an overwrite so that the block can catch up.  (Coarser than the
reference, which hands out the surviving part of a span.)
"""
import os
import threading
import time
from copy import deepcopy

import numpy as np

from bifrost_b200 import affinity, device
from bifrost_b200.ndarray import memset_array
from bifrost_b200.proclog import ProcLog
from bifrost_b200.memory import space_accessible
from bifrost_b200.ring import (Ring, ViewRing, Span, Sequence, PipelineAborted,      # noqa: F401
                               frame_axis as _frame_axis, slice_frames as _slice_frames)

_tls = threading.local()


def get_default_pipeline():
    if not hasattr(_tls, 'pipeline_stack'):
        _tls.pipeline_stack = [Pipeline()]
    return _tls.pipeline_stack[-1]


def _scope_stack():
    if not hasattr(_tls, 'scope_stack'):
        _tls.scope_stack = [{}]
    return _tls.scope_stack


class block_scope(object):
    """Attribute scope inherited by blocks created inside it (gulp_nframe,
    buffer_nframe, buffer_factor, core, gpu, share_temp_storage, fuse) --
    pipeline.py:84-134.  ``gpu`` selects the device of the blocks' threads,
    ``core`` the CPU core they are bound to, ``buffer_nframe`` /
    ``buffer_factor`` size the blocks' output rings, ``fuse=True`` collapses
    chains that have a fused kernel into one launch (Pipeline._fuse_chains).
    ``share_temp_storage`` is accepted and has no effect (the ops own their
    workspaces)."""

    def __init__(self, **kwargs):
        self.kwargs = kwargs

    def __enter__(self):
        merged = dict(_scope_stack()[-1])
        merged.update(self.kwargs)
        _scope_stack().append(merged)
        return self

    def __exit__(self, *exc):
        _scope_stack().pop()


class Pipeline(object):
    def __init__(self, name=None, **kwargs):
        self.name = name or 'Pipeline'
        self.blocks = []
        self.kwargs = kwargs
        self._abort = threading.Event()
        self._errors = []

    def __enter__(self):
        if not hasattr(_tls, 'pipeline_stack'):
            _tls.pipeline_stack = [Pipeline()]
        _tls.pipeline_stack.append(self)
        return self

    def __exit__(self, *exc):
        _tls.pipeline_stack.pop()

    def _rings(self):
        rings = []
        for b in self.blocks:
            for r in list(b.orings) + list(b.irings):
                root = r.root()
                if root not in rings:
                    rings.append(root)
        return rings

    def run(self):
        """One thread per block; returns when every block has finished."""
        self._fuse_chains()
        self._abort.clear()
        self._errors = []
        for ring in self._rings():
            ring.set_abort_event(self._abort)
        for b in self.blocks:                  # readers exist before any writer starts
            b._readers = [r.open_reader(b) for r in b.irings]
        # a block without gpu= works on the device that is current where run() is
        # called (a new thread would otherwise start on device 0)
        try:
            self._default_gpu = int(device.get_device())
        except Exception:
            self._default_gpu = None            # no CUDA device: system-space pipelines
        threads = [threading.Thread(target=self._run_block, args=(b,), name=b.name, daemon=True) for b in self.blocks]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if self._errors:
            raise self._errors[0]

    def _run_block(self, block):
        try:
            if block.core is not None:
                core = block.core if isinstance(block.core, int) else block.core[0]
                try:
                    affinity.set_core(int(core))
                except RuntimeError:            # a core this machine does not have
                    pass
            # the status logs the reference's executor keeps per block (pipeline.py:346-364,445-451)
            block._log('bind', {'ncore': 1, 'core0': affinity.get_core()})
            block._log('in', dict([('nring', len(block.irings))] +
                                  [(f'ring{i}', r.name) for i, r in enumerate(block.irings)]))
            block._log('out', dict([('nring', len(block.orings))] +
                                   [(f'ring{i}', r.name) for i, r in enumerate(block.orings)]))
            if block.gpu is not None:
                device.set_device(block.gpu)
            elif getattr(self, '_default_gpu', None) is not None:
                device.set_device(self._default_gpu)
            block.main()
        except PipelineAborted:
            pass
        except BaseException as e:             # noqa: BLE001 -- re-raised by run()
            self._errors.append(e)
            self._abort.set()
            for ring in self._rings():
                ring.wake()

    def _fuse_chains(self):
        """Honours ``block_scope(fuse=True)`` (pipeline.py:84-134 of the reference,
        where the flag only removes the ring between blocks): a chain
            transpose(['time','pol','freq','fine_time']) -> fft('fine_time', apply_fftshift=True)
            -> detect('stokes') -> [merge_axes('freq', ...)] -> reduce('freq', f) -> accumulate(n)
        whose blocks were all created under fuse=True, each feeding only the next,
        is replaced by one SpectrometerBlock (one kernel launch per gulp,
        bfSpectrometerFused) between the chain's input and output rings; and a
        correlate(...) feeding only a convert_visibilities(..., 'storage'), both
        created under fuse=True, by one correlate(..., output='storage')
        (bfLinAlgCorrelateToStorage: the same output bits, one HBM pass fewer);
        and a beamform(w) -> detect(mode) -> reduce('time', nint, op='sum'),
        mode scalar / stokes / stokes_i / coherence, each feeding only the
        next, by one beamform(w, detect=mode, nint=nint)
        (bfLinAlgBeamformDetect: the same output bits and header, one kernel)."""
        from bifrost_b200.blocks.transpose import TransposeBlock
        from bifrost_b200.blocks.fft import FftBlock
        from bifrost_b200.blocks.detect import DetectBlock
        from bifrost_b200.blocks.reduce import ReduceBlock
        from bifrost_b200.blocks.accumulate import AccumulateBlock
        from bifrost_b200.blocks.spectrometer import SpectrometerBlock
        from bifrost_b200.blocks.correlate import CorrelateBlock
        from bifrost_b200.blocks.convert_visibilities import ConvertVisibilitiesBlock
        from bifrost_b200.blocks.beamform import BeamformBlock, DETECT_MODES
        if not hasattr(_tls, 'pipeline_stack'):
            _tls.pipeline_stack = [Pipeline()]

        def only_consumer(ring, through_views=False):
            """The single block reading `ring` (optionally through one header view)."""
            if len(ring.consumers) == 1 and not ring.views:
                return ring.consumers[0]
            if through_views and not ring.consumers and len(ring.views) == 1:
                return only_consumer(ring.views[0])
            return None

        for t in [b for b in self.blocks if isinstance(b, TransposeBlock) and b.fuse]:
            if list(t.specified_axes) != ['time', 'pol', 'freq', 'fine_time']:
                continue
            f = only_consumer(t.orings[0])
            if not (isinstance(f, FftBlock) and f.fuse and f.specified_axes == ['fine_time'] and f.apply_fftshift
                    and not f.inverse and not f.real_output):
                continue
            d = only_consumer(f.orings[0])
            if not (isinstance(d, DetectBlock) and d.fuse and d.mode == 'stokes' and d.specified_axis in (None, 'pol')):
                continue
            r = only_consumer(d.orings[0], through_views=True)
            if not (isinstance(r, ReduceBlock) and r.fuse and r.specified_axis == 'freq' and r.op == 'sum'
                    and r.specified_factor in (1, 2, 4, 8, 16, 32)):
                continue
            a = only_consumer(r.orings[0])
            if not (isinstance(a, AccumulateBlock) and a.fuse and a.dtype in (None, 'f32')):
                continue
            iring, oring = t.irings[0], a.orings[0]
            _tls.pipeline_stack.append(self)
            try:
                spec = SpectrometerBlock(iring, f_avg=r.specified_factor, n_int=a.nframe,
                                         gulp_nframe=t.gulp_nframe, gpu=t.gpu, core=t.core)
            finally:
                _tls.pipeline_stack.pop()
            iring.consumers.remove(t)
            spec.orings = [oring]
            oring.owner = spec
            for b in (t, f, d, r, a):
                self.blocks.remove(b)

        # correlate -> convert_visibilities('storage'): one CorrelateBlock(output='storage'),
        # which writes the Stokes storage layout from the correlator (the same bits)
        for c in [b for b in self.blocks if isinstance(b, CorrelateBlock) and b.fuse and b.output == 'matrix']:
            v = only_consumer(c.orings[0])
            if not (isinstance(v, ConvertVisibilitiesBlock) and v.fuse and v.ofmt == 'storage'):
                continue
            iring, oring = c.irings[0], v.orings[0]
            _tls.pipeline_stack.append(self)
            try:
                corr = CorrelateBlock(iring, c.nframe_per_integration, output='storage',
                                      gulp_nframe=c.gulp_nframe, gpu=c.gpu, core=c.core)
            finally:
                _tls.pipeline_stack.pop()
            iring.consumers.remove(c)
            corr.orings = [oring]
            oring.owner = corr
            for b in (c, v):
                self.blocks.remove(b)

        # beamform -> detect -> reduce('time', nint): one BeamformBlock(detect=mode, nint=nint)
        for bm in [b for b in self.blocks if isinstance(b, BeamformBlock) and b.fuse and b.detect is None]:
            d = only_consumer(bm.orings[0])
            if not (isinstance(d, DetectBlock) and d.fuse and d.mode in DETECT_MODES
                    and d.specified_axis in (None, 'pol')):
                continue
            r = only_consumer(d.orings[0])
            if not (isinstance(r, ReduceBlock) and r.fuse and r.specified_axis in ('time', 0) and r.op == 'sum'
                    and isinstance(r.specified_factor, int) and r.specified_factor >= 2):
                continue
            iring, oring = bm.irings[0], r.orings[0]
            _tls.pipeline_stack.append(self)
            try:
                fused = BeamformBlock(iring, bm.weights, detect=d.mode, nint=r.specified_factor,
                                      gulp_nframe=bm.gulp_nframe, gpu=bm.gpu, core=bm.core)
            finally:
                _tls.pipeline_stack.pop()
            iring.consumers.remove(bm)
            fused.orings = [oring]
            oring.owner = fused
            for b in (bm, d, r):
                self.blocks.remove(b)

    def shutdown(self):
        """Stops every block at its next ring call; run() then returns."""
        self._abort.set()
        for ring in self._rings():
            ring.wake()

    def shutdown_on_signals(self, signals=None):
        """Installs handlers that shut the pipeline down (pipeline.py:271-286 of
        the reference; default SIGHUP, SIGINT, SIGQUIT, SIGTERM, SIGTSTP).  Call
        from the main thread, before run()."""
        import signal
        import warnings
        if signals is None:
            signals = [signal.SIGHUP, signal.SIGINT, signal.SIGQUIT, signal.SIGTERM, signal.SIGTSTP]

        def handler(signum, frame):
            warnings.warn(f"Received signal {signum} {signal.Signals(signum).name}, shutting down pipeline",
                          RuntimeWarning)
            self.shutdown()
        for sig in signals:
            signal.signal(sig, handler)


def _sync(*spaces):
    """The per-gulp stream synchronisation (pipeline.py:628), skipped when
    every ring involved lives in plain system memory."""
    if any(str(sp) != 'system' for sp in spaces):
        device.stream_synchronize()


PERF_LOG_PERIOD = 0.05


class Block(object):
    instance_counts = {}

    def __init__(self, irings, name=None, type_=None, **kwargs):
        self.type = type_ or self.__class__.__name__
        cnt = Block.instance_counts.get(self.type, 0)
        Block.instance_counts[self.type] = cnt + 1
        self.name = name or f"{self.type}_{cnt}"
        scope = dict(_scope_stack()[-1])
        scope.update(kwargs)
        self.gulp_nframe = scope.get('gulp_nframe')
        self.buffer_nframe = scope.get('buffer_nframe')
        self.buffer_factor = scope.get('buffer_factor')
        self.core = scope.get('core')
        self.gpu = scope.get('gpu')
        self.fuse = scope.get('fuse', False)
        self.guarantee = scope.get('guarantee', True)
        self.pipeline = get_default_pipeline()
        self.pipeline.blocks.append(self)
        self.irings = [r.orings[0] if hasattr(r, 'orings') else r for r in irings]
        for r in self.irings:
            r.consumers.append(self)
        self.orings = []
        self._readers = []
        self._proclogs = {}
        self._perf_logged = 0.

    def _log(self, kind, contents):
        """Rewrites the block's status log `<name>/<kind>` (created on first use;
        a log that cannot be written never stops the block).  The per-gulp
        'perf' log is rewritten at most every PERF_LOG_PERIOD seconds: gulps
        take well under a millisecond here, the tools that read the logs poll
        about once a second."""
        try:
            log = self._proclogs.get(kind)
            if log is None:
                log = self._proclogs[kind] = ProcLog(f"{self.name}/{kind}")
            elif kind == 'perf':
                now = time.time()
                if now - self._perf_logged < PERF_LOG_PERIOD:
                    return
                self._perf_logged = now
            log.update(contents)
        except Exception:                       # noqa: BLE001
            pass

    def create_ring(self, space):
        ring = Ring(space, self)
        ring.buffer_nframe, ring.buffer_factor = self.buffer_nframe, self.buffer_factor
        return ring

    def get_temp_storage(self, space):
        return None

    def main(self):
        raise NotImplementedError


class SourceBlock(Block):
    def __init__(self, sourcenames, gulp_nframe, space=None, *args, **kwargs):
        super(SourceBlock, self).__init__([], *args, gulp_nframe=gulp_nframe, **kwargs)
        self.sourcenames = sourcenames
        self.orings = [self.create_ring(space=space or 'system')]
        self._seq_count = 0

    def create_reader(self, sourcename):
        raise NotImplementedError

    def on_sequence(self, reader, sourcename):
        raise NotImplementedError

    def on_data(self, reader, ospans):
        raise NotImplementedError

    def main(self):
        ring = self.orings[0]
        try:
            for sourcename in self.sourcenames:
                with self.create_reader(sourcename) as reader:
                    ohdrs = self.on_sequence(reader, sourcename)
                    for ohdr in ohdrs:
                        ohdr.setdefault('time_tag', self._seq_count)
                        ohdr.setdefault('name', f"unnamed-sequence-{self._seq_count}")
                        ohdr.setdefault('gulp_nframe', self.gulp_nframe)
                    self._seq_count += 1
                    st = ring.begin_sequence(ohdrs[0], self.gulp_nframe)
                    try:
                        self._log('sequence0', ohdrs[0])
                        while True:
                            t0 = time.time()
                            ospan = ring.reserve(st, self.gulp_nframe)
                            t1 = time.time()
                            n = self.on_data(reader, [ospan])[0]
                            ring.commit(st, n)
                            self._log('perf', {'acquire_time': -1, 'reserve_time': t1 - t0,
                                               'process_time': time.time() - t1})
                            if n == 0 or n < ospan.nframe:
                                break
                    finally:
                        ring.end_sequence(st)
        finally:
            ring.end_writing()


class _ConsumerMixin(object):
    """Input side shared by transform and sink blocks: one reader on the input
    ring, spans of gulp + overlap frames advanced gulp by gulp."""

    def _check_space(self):
        valid = self.define_valid_input_spaces()
        if valid != 'any' and not any(space_accessible(self.irings[0].space, [s]) for s in valid):
            raise ValueError(f"{self.name}: input space '{self.irings[0].space}' not in {valid}")

    def _gulp(self, iseq):
        return self.gulp_nframe or iseq.header.get('gulp_nframe') or 1

    def main(self):
        reader = self._readers[0]
        try:
            for st, iseq in reader.sequences():
                self._check_space()
                overlap = self._open_sequence(iseq)
                gulp = self._gulp(iseq)
                self._ist = st
                reader.open(st, gulp, overlap)
                try:
                    self._begin_outputs(iseq, gulp, overlap)
                    self._log('sequence0', iseq.header)
                    offset = 0
                    force_skip = False
                    while True:
                        t0 = time.time()
                        ispan = reader.acquire(st, iseq, offset, gulp + overlap)
                        # (an unguaranteed reader that was lapped gets an empty span
                        # and the number of frames it lost)
                        nframe = ispan.nframe + ispan.nframe_skipped
                        if nframe <= overlap:                  # nothing new (or nothing at all)
                            break
                        t1 = time.time()
                        self._reserve_time = 0.
                        skip = force_skip or ispan.nframe_skipped > 0
                        self._process(ispan, overlap, nframe, skip)
                        if not reader.guarantee:
                            # frames that were overwritten while on_data worked on them are
                            # void too; one more gulp is then dropped so that a block that
                            # fell behind can catch up (pipeline.py:630-643 of the reference)
                            force_skip = (not skip) and ispan.nframe_overwritten > 0
                        self._log('perf', {'acquire_time': t1 - t0, 'reserve_time': self._reserve_time,
                                           'process_time': time.time() - t1 - self._reserve_time})
                        offset += gulp
                        reader.release(st, offset)
                        if nframe < gulp + overlap:            # ragged final gulp
                            break
                    self.on_sequence_end(iseq)
                finally:
                    self._end_outputs()
                    reader.close(st)
        finally:
            self._stop_outputs()


class TransformBlock(_ConsumerMixin, Block):
    def __init__(self, iring, *args, **kwargs):
        super(TransformBlock, self).__init__([iring], *args, **kwargs)
        self.iring = self.irings[0]
        self.orings = [self.create_ring(space=self.iring.space)]
        self._ost = None

    # ---- user hooks (same names/meaning as pipeline.py:703-748)
    def define_valid_input_spaces(self):
        return 'any'

    def define_input_overlap_nframe(self, iseq):
        return 0

    def define_output_nframes(self, input_nframe):
        return input_nframe

    def on_sequence(self, iseq):
        raise NotImplementedError

    def on_sequence_end(self, iseq):
        pass

    def on_data(self, ispan, ospan):
        raise NotImplementedError

    def on_skip(self, islice, ospan):
        memset_array(ospan.data, 0)

    # ---- executor internals
    def _open_sequence(self, iseq):
        self._ohdr = self.on_sequence(iseq)
        self._ohdr.setdefault('gulp_nframe', iseq.header.get('gulp_nframe'))
        return self.define_input_overlap_nframe(iseq)

    def _begin_outputs(self, iseq, gulp, overlap):
        self._ost = self.orings[0].begin_sequence(self._ohdr, self.define_output_nframes(gulp + overlap))

    def _process(self, ispan, overlap, nframe=None, skip=False):
        ring = self.orings[0]
        onframe = self.define_output_nframes(ispan.nframe if nframe is None else nframe)
        # a block that commits rarely (accumulate) is handed the same frames again
        t0 = time.time()
        ospan = ring.reserve(self._ost, onframe)
        self._reserve_time = time.time() - t0
        ncommit = None
        if not skip:
            ncommit = self.on_data(ispan, ospan)
            if not self._readers[0].guarantee:
                _sync(self.irings[0].space, ring.space)        # the kernels have read what they will read
                if ispan.nframe_overwritten:
                    skip = True
        if skip:
            # the frames were lost to the writer: the output keeps its cadence, with
            # whatever on_skip puts there (zeros)
            lost = ispan.nframe if nframe is None else nframe
            self.on_skip(slice(ispan.frame_offset, ispan.frame_offset + lost), ospan)
            ncommit = None
        if ncommit is None:
            ooverlap = self.define_output_nframes(overlap) if overlap else 0
            ncommit = max(onframe - ooverlap, 0)
        if str(ring.space) == 'system':
            _sync(self.irings[0].space)        # (commit synchronises for device rings)
        ring.commit(self._ost, ncommit)

    def _end_outputs(self):
        if self._ost is not None:
            self.orings[0].end_sequence(self._ost)
            self._ost = None

    def _stop_outputs(self):
        self.orings[0].end_writing()


class SinkBlock(_ConsumerMixin, Block):
    def __init__(self, iring, *args, **kwargs):
        super(SinkBlock, self).__init__([iring], *args, **kwargs)
        self.iring = self.irings[0]

    def define_valid_input_spaces(self):
        return 'any'

    def define_input_overlap_nframe(self, iseq):
        return 0

    def on_sequence(self, iseq):
        raise NotImplementedError

    def on_sequence_end(self, iseq):
        pass

    def on_data(self, ispan):
        raise NotImplementedError

    def on_skip(self, islice):
        """Frames `islice` of the sequence were lost (unguaranteed readers only)."""
        pass

    def _open_sequence(self, iseq):
        self.on_sequence(iseq)
        return self.define_input_overlap_nframe(iseq)

    def _begin_outputs(self, iseq, gulp, overlap):
        pass

    def _process(self, ispan, overlap, nframe=None, skip=False):
        if skip:
            self.on_skip(slice(ispan.frame_offset, ispan.frame_offset + (nframe or 0)))
            return
        self.on_data(ispan)
        _sync(self.irings[0].space)

    def _end_outputs(self):
        pass

    def _stop_outputs(self):
        pass


class BlockView(object):
    """What ``block_view`` returns: usable wherever a block is accepted as an
    input (it only carries an output ring)."""

    def __init__(self, ring, base):
        self.orings = [ring]
        self.base = base


def block_view(block, header_transform):
    """A view of `block` whose output header is passed through
    `header_transform(hdr) -> hdr` (pipeline.py:block_view); no data moves:
    readers of the view read the parent ring's storage."""
    parent = block.orings[0]
    ring = ViewRing(parent, header_transform)
    parent.views.append(ring)
    return BlockView(ring, block)
