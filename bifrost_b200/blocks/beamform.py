"""beamform block: ['time','freq','station','pol'] voltages -> ['time','freq','beam']
cf32 beams, beam[t] = sum_k w[k] x[t][k] over k = (station, pol), with no
conjugation (as the reference's beamformer kernel).  Callers who want conj(w)
pass it.  The data path is one bfLinAlgMatMul per gulp, which runs the sm_90a
beamformer (csrc/beamform.cu) for ci4 / ci8 voltages."""
import numpy as np

from bifrost_b200.pipeline import TransformBlock
from bifrost_b200.linalg import LinAlg
from bifrost_b200.blocks import _header as H
from bifrost_b200.ndarray import ndarray, asarray

_IN_AXES = ['time', 'freq', 'station', 'pol']
_IN_DTYPES = ('ci4', 'ci8', 'ci16', 'cf32')


class BeamformBlock(TransformBlock):
    def __init__(self, iring, weights, *args, **kwargs):
        """weights: complex [freq, beam, station, pol], numpy or a bf ndarray."""
        super(BeamformBlock, self).__init__(iring, *args, **kwargs)
        if isinstance(weights, ndarray) and weights.bf.space != 'system':
            weights = weights.copy('system')
        self.weights = np.asarray(weights)
        if not np.iscomplexobj(self.weights) or self.weights.ndim != 4:
            raise ValueError("weights must be complex [freq, beam, station, pol], got %s %s"
                             % (self.weights.dtype, self.weights.shape))
        self.linalg = LinAlg()
        self.d_w = None

    def define_valid_input_spaces(self):
        return ('cuda',)

    def on_sequence(self, iseq):
        ihdr = iseq.header
        itensor = ihdr['_tensor']
        if itensor['labels'] != _IN_AXES:
            raise ValueError("Expected axes %s, got %s" % (_IN_AXES, itensor['labels']))
        if itensor['dtype'] not in _IN_DTYPES:
            raise ValueError("Expected one of %s voltages, got %s" % (_IN_DTYPES, itensor['dtype']))
        nchan, nstand, npol = itensor['shape'][1:]
        nfreq_w, nbeam, nstand_w, npol_w = self.weights.shape
        if (nfreq_w, nstand_w, npol_w) != (nchan, nstand, npol):
            raise ValueError("weights of shape %s do not match [freq=%i, beam, station=%i, pol=%i]"
                             % (self.weights.shape, nchan, nstand, npol))
        # cf32 [freq, beam, station*pol]; copied to the device once, by the
        # sequence's first gulp
        self.w = np.ascontiguousarray(self.weights.reshape(nchan, nbeam, nstand * npol), dtype=np.complex64)
        self.d_w = None
        ohdr, otensor = H.derive(ihdr)
        otensor['dtype'] = 'cf32'
        # [time, freq, station, pol] -> [time, freq, beam]
        H.remap_axes(itensor, otensor, [0, 1, 2])
        otensor['shape'] = [-1, nchan, nbeam]
        otensor['labels'] = ['time', 'freq', 'beam']
        if 'scales' in otensor:
            otensor['scales'][2] = None
        if 'units' in otensor:
            otensor['units'][2] = None
        return ohdr

    def on_data(self, ispan, ospan):
        if self.d_w is None:
            self.d_w = asarray(self.w, space='cuda')
        idata, odata = ispan.data, ospan.data
        ntime, nchan, nstand, npol = idata.shape
        # a = w [freq, beam, K]; b = x as [freq, K, time]; c = out as [freq, beam, time]
        x = idata.reshape(ntime, nchan, nstand * npol).transpose(1, 2, 0)
        c = odata.transpose(1, 2, 0)
        self.linalg.matmul(1., self.d_w, x, 0., c)


def beamform(iring, weights, *args, **kwargs):
    """Form beams from ['time','freq','station','pol'] voltages with complex
    weights [freq, beam, station, pol]: out[t, f, b] = sum_{s,p} w[f, b, s, p] x[t, f, s, p]."""
    return BeamformBlock(iring, weights, *args, **kwargs)
