"""detect block (same contract as python/bifrost/blocks/detect.py:38-160).  The
reference builds bfMap strings; this build calls the fixed kernels directly
(bfDetect) -- the strings are still accepted by bf.map (csrc/map.cu)."""
from bifrost_b200.pipeline import TransformBlock
from bifrost_b200.DataType import DataType
from bifrost_b200.map import detect as bf_detect
from bifrost_b200.blocks import _header as H

# output length of a 2-long pol axis per mode (absent: unchanged)
_POL_OUT = {'stokes': 4, 'coherence': 4, 'stokes_i': 1}


def _pol_axis(tensor, mode, axis):
    """The axis the Jones / Stokes products run over, or None (scalar)."""
    if axis is None:
        if 'labels' not in tensor:
            raise TypeError("Polarization (pol) index must be labelled, or axis must be set manually")
        if mode != 'scalar' and 'pol' in tensor['labels']:
            return tensor['labels'].index('pol')
        return None
    return H.axis_index(tensor, axis)


def detect_header(ihdr, mode, axis=None):
    """(ohdr, pol axis or None, npol) of detect(mode, axis) on a sequence with
    header ihdr; also the header of beamform(..., detect=mode)."""
    ohdr, otensor = H.derive(ihdr)
    itype = DataType(otensor['dtype'])
    if not itype.is_complex:
        raise TypeError("Input data must be complex")
    pol = _pol_axis(otensor, mode, axis)
    npol = 1
    if pol is not None:
        npol = otensor['shape'][pol]
        if npol not in (1, 2):
            raise ValueError("Axis must have length 1 or 2")
        if npol == 2:
            otensor['shape'][pol] = _POL_OUT.get(mode, 2)
        if 'labels' in otensor:
            otensor['labels'][pol] = 'pol'
    # only a 2-pol Jones product stays complex
    otype = itype if (mode == 'jones' and npol == 2) else itype.as_real()
    otensor['dtype'] = str(otype.as_floating_point())
    return ohdr, pol, npol


class DetectBlock(TransformBlock):
    def __init__(self, iring, mode, axis=None, *args, **kwargs):
        super(DetectBlock, self).__init__(iring, *args, **kwargs)
        self.specified_axis = axis
        self.mode = mode.lower()

    def define_valid_input_spaces(self):
        return ('cuda',)

    def on_sequence(self, iseq):
        ohdr, self.axis, self.npol = detect_header(iseq.header, self.mode, self.specified_axis)
        return ohdr

    def on_data(self, ispan, ospan):
        if self.npol == 1:
            bf_detect(ispan.data, ospan.data, 'scalar')
        else:
            bf_detect(ispan.data, ospan.data, self.mode, self.axis)


def detect(iring, mode, axis=None, *args, **kwargs):
    """Square-law detection: 'scalar', 'jones', 'stokes', 'stokes_i', 'coherence'."""
    return DetectBlock(iring, mode, axis, *args, **kwargs)
