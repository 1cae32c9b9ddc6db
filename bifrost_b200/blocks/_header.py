"""Small helpers the blocks share for rewriting sequence headers.  A `_tensor`
entry describes the stream: dtype, shape (-1 marks the frame axis), and per-axis
labels / scales / units (any of which may be absent)."""
from copy import deepcopy

from bifrost_b200.units import convert_units

PER_AXIS = ('shape', 'labels', 'scales', 'units')


def derive(ihdr):
    """Output header that starts out as a deep copy of the input's."""
    ohdr = deepcopy(ihdr)
    return ohdr, ohdr['_tensor']


def axis_index(tensor, axis):
    """An axis given by label or by position."""
    return tensor['labels'].index(axis) if isinstance(axis, str) else axis


def frame_axis(tensor):
    return tensor['shape'].index(-1)


def check_dtype(tensor, dtypes, op, noun):
    """TypeError unless the stream's dtype is one of `dtypes`."""
    if tensor['dtype'] not in dtypes:
        raise TypeError("%s takes %s %s, got %s" % (op, '/'.join(dtypes), noun, tensor['dtype']))


def check_time_frames(tensor, dtypes, op, noun):
    """Refuses a stream that is not [..., 'time'] with time as the frame axis
    (KeyError) or whose dtype is not one of `dtypes` (TypeError)."""
    if tensor['shape'][-1] != -1 or tensor.get('labels', [None])[-1] != 'time':
        raise KeyError("Expected axes [..., 'time'] with time as the frame axis, got %s" % tensor.get('labels'))
    check_dtype(tensor, dtypes, op, noun)


def channel_band(ihdr, dtypes, op, noun):
    """(tensor, nchan, f0 MHz, df MHz, tsamp s) of a ['freq', ..., 'time']
    header with time as the frame axis and a dtype in `dtypes`; KeyError or
    TypeError otherwise.  tsamp keeps the sign of the time step."""
    t = ihdr['_tensor']
    labels = list(t.get('labels') or [])
    if len(labels) < 2 or labels[0] != 'freq' or labels[-1] != 'time' or t['shape'][-1] != -1:
        raise KeyError("Expected axes ['freq', ..., 'time'] with time as the frame axis, got %s" % labels)
    check_dtype(t, dtypes, op, noun)
    funit, tunit = t['units'][0], t['units'][-1]
    f0 = convert_units(t['scales'][0][0], funit, 'MHz')
    df = convert_units(t['scales'][0][1], funit, 'MHz')
    tsamp = convert_units(t['scales'][-1][1], tunit, 's')
    return t, t['shape'][0], f0, df, tsamp


def remap_axes(itensor, otensor, picks):
    """otensor's per-axis lists become [itensor[...][i] for i in picks] (a pick
    may repeat: each occurrence gets its own copy)."""
    for key in PER_AXIS:
        if key in itensor:
            otensor[key] = [deepcopy(itensor[key][i]) for i in picks]


def scale_step(tensor, axis, factor):
    """Multiplies the sampling step of `axis` (scales = [origin, step])."""
    if 'scales' in tensor and tensor['scales'][axis] is not None:
        origin, step = tensor['scales'][axis]
        tensor['scales'][axis] = [origin, step * factor]
