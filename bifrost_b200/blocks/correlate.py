"""correlate block (same contract as python/bifrost/blocks/correlate.py:37-138;
the data path is bfLinAlgMatMul(a=NULL, b=x), or bfLinAlgCorrelateCi4 for ci4:
the int8 tensor-core correlator).

output='storage' (extension) emits what convert_visibilities(..., 'storage')
would make of the matrix output, bit for bit and with the same header, from
bfLinAlgCorrelateToStorage: one kernel per integration when an integration is
one gulp."""
from bifrost_b200.pipeline import TransformBlock
from bifrost_b200.linalg import LinAlg
from bifrost_b200.blocks import _header as H
from bifrost_b200.blocks.convert_visibilities import matrix_to_storage_header
from bifrost_b200 import visibilities
from bifrost_b200.ndarray import empty

_IN_AXES = ['time', 'freq', 'station', 'pol']


class CorrelateBlock(TransformBlock):
    def __init__(self, iring, nframe_per_integration, output='matrix', *args, **kwargs):
        super(CorrelateBlock, self).__init__(iring, *args, **kwargs)
        if output not in ('matrix', 'storage'):
            raise ValueError("output must be 'matrix' or 'storage', got %r" % (output,))
        self.nframe_per_integration = nframe_per_integration
        self.output = output
        self.linalg = LinAlg()
        self._acc = None            # storage output over several gulps: C is summed here

    def define_valid_input_spaces(self):
        return ('cuda',)

    def define_output_nframes(self, input_nframe):
        return 1

    def on_sequence(self, iseq):
        self.nframe_integrated = 0
        ihdr = iseq.header
        if ihdr['_tensor']['labels'] != _IN_AXES:
            raise ValueError("Expected axes %s, got %s" % (_IN_AXES, ihdr['_tensor']['labels']))
        ohdr, otensor = H.derive(ihdr)
        otensor['dtype'] = 'cf32'
        # [time, freq, station, pol] -> [time, freq, station_i, pol_i, station_j, pol_j]
        H.remap_axes(ihdr['_tensor'], otensor, [0, 1, 2, 3, 2, 3])
        otensor['labels'] = ['time', 'freq', 'station_i', 'pol_i', 'station_j', 'pol_j']
        H.scale_step(otensor, 0, self.nframe_per_integration)
        ohdr['matrix_fill_mode'] = 'lower'
        # an integration is made of whole input gulps: the gulp the block reads
        # (its own setting, else the upstream one, capped at one integration) has
        # to divide nframe_per_integration (blocks/correlate.py:67-74)
        ohdr['gulp_nframe'] = min(ihdr.get('gulp_nframe') or 1, self.nframe_per_integration)
        gulp = self.gulp_nframe or ohdr['gulp_nframe']
        if self.nframe_per_integration % gulp:
            raise ValueError("gulp_nframe (%i) does not divide nframe_per_integration (%i)"
                             % (gulp, self.nframe_per_integration))
        if self.output == 'storage':
            matrix_to_storage_header(ohdr)
        return ohdr

    def _gulp(self, iseq):
        # the input is read in gulps that tile an integration
        return self.gulp_nframe or min(iseq.header.get('gulp_nframe') or 1, self.nframe_per_integration)

    def on_data(self, ispan, ospan):
        idata, odata = ispan.data, ospan.data
        ntime, nchan, nstand, npol = idata.shape
        n = nstand * npol
        # [time, freq, stand*pol] -> [freq, time, stand*pol] view; out [freq, n, n]
        x = idata.reshape(ntime, nchan, n).transpose(1, 0, 2)
        first = self.nframe_integrated == 0
        done = self.nframe_integrated + ispan.nframe == self.nframe_per_integration
        if self.output == 'matrix':
            self.linalg.matmul(1., None, x, 0. if first else 1., odata.reshape(nchan, n, n))
        elif first and done:
            self.linalg.correlate_to_storage(x, odata.reshape(odata.shape[1:]))
        else:
            # the matrix block's sum, in a private buffer: an output frame holds Stokes only
            if self._acc is None or self._acc.shape != (nchan, n, n):
                self._acc = empty((nchan, n, n), dtype='cf32', space='cuda')
            self.linalg.matmul(1., None, x, 0. if first else 1., self._acc)
            if done:
                visibilities.to_storage(self._acc.reshape(nchan, nstand, npol, nstand, npol),
                                        odata.reshape(odata.shape[1:]))
        self.nframe_integrated += ispan.nframe
        if self.nframe_integrated > self.nframe_per_integration:
            raise RuntimeError("integration overran: gulp does not tile nframe_per_integration")
        if done:
            self.nframe_integrated = 0
            return 1
        return 0


def correlate(iring, nframe_per_integration, *args, **kwargs):
    """Cross-multiply ['time','freq','station','pol'] voltages into lower-triangular
    visibilities ['time','freq','station_i','pol_i','station_j','pol_j'], or with
    output='storage' into ['time','baseline','freq','stokes'] (the layout of
    convert_visibilities(..., 'storage'), npol = 2).  The voltages may be ci4
    (high nibble real), ci8, ci16 or cf32; ci4 gives the bytes of the same
    pipeline on ci8 with the same values, without an unpack pass (the tensor
    cores read it when station x pol is a multiple of 16)."""
    return CorrelateBlock(iring, nframe_per_integration, *args, **kwargs)
