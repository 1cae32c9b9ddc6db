"""reduce block (same contract as python/bifrost/blocks/reduce.py:38-118; the
data path is bfReduce)."""
from bifrost_b200.pipeline import TransformBlock
from bifrost_b200.reduce import reduce as bf_reduce
from bifrost_b200.blocks import _header as H

_COMPLEX_IN = ('cf32', 'ci8', 'ci16')


def reduce_header(ihdr, axis, factor=None, op='sum'):
    """(ohdr, axis index, factor, frame factor) of reduce(axis, factor, op) on a
    sequence with header ihdr; also the header of beamform(..., nint=factor)."""
    ohdr, otensor = H.derive(ihdr)
    # power ops give real output; plain ops keep complex input complex
    keeps_complex = ihdr['_tensor']['dtype'] in _COMPLEX_IN and not op.startswith('pwr')
    otensor['dtype'] = 'cf32' if keeps_complex else 'f32'
    axis = H.axis_index(otensor, axis)
    frame_factor = 1
    if axis == H.frame_axis(otensor):
        # along time: fewer frames come out, the shape entry stays -1
        if factor is None:
            raise ValueError("Cannot reduce all of the frame axis")
        frame_factor = factor
        ohdr['gulp_nframe'] = max((ihdr.get('gulp_nframe') or factor) // factor, 1)
    else:
        length = otensor['shape'][axis]
        if factor is None:
            factor = length
        if length % factor:
            raise ValueError("Reduce factor does not divide axis length")
        otensor['shape'][axis] = length // factor
    H.scale_step(otensor, axis, factor)
    return ohdr, axis, factor, frame_factor


class ReduceBlock(TransformBlock):
    def __init__(self, iring, axis, factor=None, op='sum', *args, **kwargs):
        super(ReduceBlock, self).__init__(iring, *args, **kwargs)
        self.specified_axis = axis
        self.specified_factor = factor
        self.op = op

    def define_valid_input_spaces(self):
        return ('cuda',)

    def define_output_nframes(self, input_nframe):
        return input_nframe // self.frame_factor

    def on_sequence(self, iseq):
        ohdr, self.axis, self.factor, self.frame_factor = reduce_header(
            iseq.header, self.specified_axis, self.specified_factor, self.op)
        return ohdr

    def on_data(self, ispan, ospan):
        bf_reduce(ispan.data, ospan.data, self.op)


def reduce(iring, axis, factor=None, op='sum', *args, **kwargs):
    """Reduce `axis` by `factor` (None = all) with op sum/mean/min/max/stderr/pwr*."""
    return ReduceBlock(iring, axis, factor, op, *args, **kwargs)
