"""pulse_search block: boxcar matched-filter search of a dispersion stream
(extension, bfPulseSearch*; no reference counterpart)."""
from bifrost_b200.pipeline import TransformBlock
from bifrost_b200.pulse_search import PulseSearch, output_nblock
from bifrost_b200.blocks import _header as H

DEFAULT_WIDTHS = (1, 2, 4, 8, 16, 32, 64, 128, 256)
PEAK_FIELDS = ['snr', 'offset', 'width']


def pulse_search_header(ihdr, widths, decim):
    """Output header of pulse_search(widths, decim) on a [..., trial, 'time']
    f32 sequence with header ihdr: the time axis (still the frame axis) steps
    by decim samples and a last 'peak' axis of length 3 holds PEAK_FIELDS.
    `peak_decim` is decim, so a consumer can turn a frame and an offset back
    into a sample of the searched series."""
    ohdr, t = H.derive(ihdr)
    H.check_time_frames(t, ('f32',), 'pulse_search', 'input')
    H.scale_step(t, len(t['shape']) - 1, decim)
    for key, value in (('shape', 3), ('labels', 'peak'), ('scales', None), ('units', None)):
        if key in t:
            t[key].append(value)
    ohdr.update(boxcar_widths=[int(w) for w in widths], peak_fields=list(PEAK_FIELDS), peak_decim=int(decim))
    return ohdr


class PulseSearchBlock(TransformBlock):
    """Each output frame is one block of `decim` start samples: per row, the
    (snr, start offset, width) of its highest-S/N boxcar.  The mean and
    standard deviation that normalise each width are those of the span the
    block was searched in: one gulp of gulp_nframe starts (plus the W - 1
    samples of look-ahead), so every block of a gulp shares them and the last,
    ragged gulp has its own."""

    def __init__(self, iring, widths=DEFAULT_WIDTHS, decim=256, *args, **kwargs):
        super(PulseSearchBlock, self).__init__(iring, *args, **kwargs)
        self.widths = [int(w) for w in widths]
        self.decim = int(decim)
        self.plan = PulseSearch()
        self.plan.init(self.widths, self.decim)
        self.overlap = max(self.widths) - 1

    def define_valid_input_spaces(self):
        return ('cuda',)

    def define_input_overlap_nframe(self, iseq):
        return self.overlap

    def define_output_nframes(self, input_nframe):
        return output_nblock(input_nframe, self.widths, self.decim)

    def on_sequence(self, iseq):
        gulp = self._gulp(iseq)
        if gulp % self.decim:
            raise ValueError("gulp_nframe (%d) must be a multiple of decim (%d)" % (gulp, self.decim))
        ohdr = pulse_search_header(iseq.header, self.widths, self.decim)
        ohdr['gulp_nframe'] = gulp // self.decim
        return ohdr

    def on_data(self, ispan, ospan):
        nblk = output_nblock(ispan.nframe, self.widths, self.decim)
        if nblk == 0:
            return 0
        self.plan.execute(ispan.data, ospan.data)
        return nblk


def pulse_search(iring, widths=DEFAULT_WIDTHS, decim=256, *args, **kwargs):
    """Boxcar pulse search of a [..., 'dispersion', 'time'] f32 stream (any
    label for the trial axis): one (snr, offset, width) peak per row and
    `decim` start samples, over boxcar `widths` (see PulseSearchBlock)."""
    return PulseSearchBlock(iring, widths, decim, *args, **kwargs)
