"""beamform block: ['time','freq','station','pol'] voltages -> ['time','freq','beam']
cf32 beams, beam[t] = sum_k w[k] x[t][k] over k = (station, pol), with no
conjugation (as the reference's beamformer kernel).  Callers who want conj(w)
pass it.  The data path is one bfLinAlgMatMul per gulp, which runs the sm_90a
beamformer (csrc/beamform.cu) for ci4 / ci8 voltages.

Weights [freq, beam, bpol=2, station, pol] form dual-polarisation beams
['time','freq','beam','pol'].  detect= makes power beams: the output is then
what detect(mode) -> reduce('time', nint) would make of the beams, bit for bit
and with the same header, from one bfLinAlgBeamformDetect per gulp."""
import numpy as np

from bifrost_b200.pipeline import TransformBlock
from bifrost_b200.linalg import LinAlg
from bifrost_b200.blocks import _header as H
from bifrost_b200.blocks.detect import detect_header
from bifrost_b200.blocks.reduce import reduce_header
from bifrost_b200.ndarray import ndarray, asarray

_IN_AXES = ['time', 'freq', 'station', 'pol']
_IN_DTYPES = ('ci4', 'ci8', 'ci16', 'cf32')
DETECT_MODES = ('scalar', 'stokes', 'stokes_i', 'coherence')


class BeamformBlock(TransformBlock):
    def __init__(self, iring, weights, detect=None, nint=1, *args, **kwargs):
        """weights: complex [freq, beam, station, pol] or [freq, beam, bpol=2,
        station, pol], numpy or a bf ndarray."""
        super(BeamformBlock, self).__init__(iring, *args, **kwargs)
        if isinstance(weights, ndarray) and weights.bf.space != 'system':
            weights = weights.copy('system')
        self.weights = np.asarray(weights)
        if not np.iscomplexobj(self.weights) or self.weights.ndim not in (4, 5) or \
                (self.weights.ndim == 5 and self.weights.shape[2] != 2):
            raise ValueError("weights must be complex [freq, beam, station, pol] or [freq, beam, 2, station, pol], "
                             "got %s %s" % (self.weights.dtype, self.weights.shape))
        if detect is not None and detect not in DETECT_MODES:
            raise ValueError("detect must be None or one of %s, got %r" % (DETECT_MODES, detect))
        if int(nint) != nint or nint < 1 or (detect is None and nint != 1):
            raise ValueError("nint must be a positive integer, and 1 without detect; got %r" % (nint,))
        self.detect = detect
        self.nint = int(nint)
        self.linalg = LinAlg()
        self.d_w = None

    def define_valid_input_spaces(self):
        return ('cuda',)

    def define_output_nframes(self, input_nframe):
        return input_nframe // self.nint

    def on_sequence(self, iseq):
        ihdr = iseq.header
        itensor = ihdr['_tensor']
        if itensor['labels'] != _IN_AXES:
            raise ValueError("Expected axes %s, got %s" % (_IN_AXES, itensor['labels']))
        if itensor['dtype'] not in _IN_DTYPES:
            raise ValueError("Expected one of %s voltages, got %s" % (_IN_DTYPES, itensor['dtype']))
        nchan, nstand, npol = itensor['shape'][1:]
        nfreq_w, nbeam = self.weights.shape[:2]
        nstand_w, npol_w = self.weights.shape[-2:]
        if (nfreq_w, nstand_w, npol_w) != (nchan, nstand, npol):
            raise ValueError("weights of shape %s do not match [freq=%i, beam, ..., station=%i, pol=%i]"
                             % (self.weights.shape, nchan, nstand, npol))
        gulp = self._gulp(iseq)
        if gulp % self.nint:
            raise ValueError("gulp_nframe (%i) is not a multiple of nint (%i)" % (gulp, self.nint))
        # cf32 [freq, beam rows, station*pol], beam rows 2j, 2j+1 the pols of
        # beam j for 5-D weights; copied to the device once, by the sequence's
        # first gulp
        self.nrow = nbeam * (2 if self.weights.ndim == 5 else 1)
        self.w = np.ascontiguousarray(self.weights.reshape(nchan, self.nrow, nstand * npol), dtype=np.complex64)
        self.d_w = None
        ohdr, otensor = H.derive(ihdr)
        otensor['dtype'] = 'cf32'
        if self.weights.ndim == 4:
            # [time, freq, station, pol] -> [time, freq, beam]
            H.remap_axes(itensor, otensor, [0, 1, 2])
            otensor['shape'] = [-1, nchan, nbeam]
            otensor['labels'] = ['time', 'freq', 'beam']
        else:
            # [time, freq, station, pol] -> [time, freq, beam, pol]
            H.remap_axes(itensor, otensor, [0, 1, 2, 3])
            otensor['shape'] = [-1, nchan, nbeam, 2]
            otensor['labels'] = ['time', 'freq', 'beam', 'pol']
        if 'scales' in otensor:
            otensor['scales'][2] = None
        if 'units' in otensor:
            otensor['units'][2] = None
        if self.detect is None:
            return ohdr
        # the headers of detect(mode) and reduce('time', nint) after it
        ohdr.setdefault('gulp_nframe', ihdr.get('gulp_nframe'))      # as the executor sets it on a ring
        ohdr, _, npol_det = detect_header(ohdr, self.detect)
        self.mode = self.detect if npol_det == 2 else 'scalar'
        if self.nint > 1:
            ohdr = reduce_header(ohdr, 'time', self.nint, 'sum')[0]
        return ohdr

    def on_data(self, ispan, ospan):
        if self.d_w is None:
            self.d_w = asarray(self.w, space='cuda')
        idata, odata = ispan.data, ospan.data
        ntime, nchan, nstand, npol = idata.shape
        nout = ntime // self.nint
        # a = w [freq, beam rows, K]; b = x as [freq, K, time]
        x = idata[:nout * self.nint].reshape(nout * self.nint, nchan, nstand * npol).transpose(1, 2, 0)
        if self.detect is None:
            # c = out as [freq, beam rows, time]
            self.linalg.matmul(1., self.d_w, x, 0., odata.reshape(ntime, nchan, self.nrow).transpose(1, 2, 0))
            return
        # out as [freq, beam rows / npb, nprod, time / nint]
        nprod = 1 if self.mode in ('scalar', 'stokes_i') else 4
        nobeam = self.nrow if self.mode == 'scalar' else self.nrow // 2
        out = odata.reshape(nout, nchan, nobeam, nprod).transpose(1, 2, 3, 0)
        self.linalg.beamform_detect(self.d_w, x, out, self.mode, self.nint)


def beamform(iring, weights, *args, **kwargs):
    """Form beams from ['time','freq','station','pol'] voltages with complex
    weights [freq, beam, station, pol]: out[t, f, b] = sum_{s,p} w[f, b, s, p] x[t, f, s, p]
    (cf32 ['time','freq','beam']), or [freq, beam, bpol, station, pol] with
    bpol = 2: cf32 ['time','freq','beam','pol'].

    detect='scalar' | 'stokes' | 'stokes_i' | 'coherence' and nint write f32
    power beams instead: what detect(mode) -> reduce('time', nint) make of
    the beams (the pol axis holds the detected products; without one every
    mode is 'scalar', as in detect), bit for bit and with the same header.
    gulp_nframe must be a multiple of nint."""
    return BeamformBlock(iring, weights, *args, **kwargs)
