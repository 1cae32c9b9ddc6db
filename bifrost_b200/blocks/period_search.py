"""period_search block: whitened, harmonic-summed power spectra of a
dispersion bank's FFTs (extension, bfPeriodSearch*; no reference counterpart).

The periodicity search of an FDMT bank cuts each DM trial's time series into
nfft-sample frames, transforms them and searches the spectra:

    d = blocks.fdmt(fil, max_delay=794, gulp_nframe=nfft)
    v = views.split_axis(d, 'time', nfft, label='fine_time')
    f = blocks.fft(v, 'fine_time', axis_labels='fft_freq')
    s = blocks.period_search(f, nharm=16, window=1024, decim=64)

Each output frame holds, per DM trial and harmonic level, the best
(power, bin offset) of every `decim` bins of one spectrum; rank peaks of
different levels with bf.period_search.significance."""
from bifrost_b200.pipeline import TransformBlock
from bifrost_b200.period_search import PeriodSearch, output_nblock, output_nlevel
from bifrost_b200.blocks import _header as H

PEAK_FIELDS = ['power', 'offset']


def period_search_header(ihdr, nharm, window, decim):
    """Output header of period_search(nharm, window, decim) on a
    [..., 'time', <freq>] cf32 sequence with header ihdr (time the frame axis,
    one spectrum per frame): a 'harmonic' axis of log2(nharm) + 1 levels goes
    in front of the freq axis, whose step grows by decim, and a last 'peak'
    axis of length 2 holds PEAK_FIELDS."""
    ohdr, t = H.derive(ihdr)
    labels = t.get('labels') or []
    if len(t['shape']) < 2 or t['shape'][-2] != -1 or len(labels) < 2 or labels[-2] != 'time':
        raise KeyError("Expected axes [..., 'time', <freq>] with time as the frame axis, got %s" % labels)
    H.check_dtype(t, ('cf32',), 'period_search', 'spectra')
    nbin = t['shape'][-1]
    fax = len(t['shape']) - 1
    H.scale_step(t, fax, decim)
    t['dtype'] = 'f32'
    t['shape'][fax] = output_nblock(nbin, decim)
    for key, harmonic, peak in (('shape', output_nlevel(nharm), 2), ('labels', 'harmonic', 'peak'),
                                ('scales', None, None), ('units', None, None)):
        if key in t:
            t[key].insert(fax, harmonic)
            t[key].append(peak)
    ohdr.update(harmonics=[1 << l for l in range(output_nlevel(nharm))],
                peak_fields=list(PEAK_FIELDS), whiten_window=int(window))
    return ohdr


class PeriodSearchBlock(TransformBlock):
    """Each output frame is the peak map of one input spectrum: per row and
    harmonic level, the (power, bin offset) of the largest harmonic sum in
    every block of `decim` bins.  Frames are independent, so there is no
    overlap and any gulp works."""

    def __init__(self, iring, nharm=16, window=1024, decim=64, *args, **kwargs):
        super(PeriodSearchBlock, self).__init__(iring, *args, **kwargs)
        self.nharm, self.window, self.decim = int(nharm), int(window), int(decim)
        self.plan = PeriodSearch()
        self.plan.init(self.nharm, self.window, self.decim)

    def define_valid_input_spaces(self):
        return ('cuda',)

    def on_sequence(self, iseq):
        return period_search_header(iseq.header, self.nharm, self.window, self.decim)

    def on_data(self, ispan, ospan):
        self.plan.execute(ispan.data, ospan.data)


def period_search(iring, nharm=16, window=1024, decim=64, *args, **kwargs):
    """Harmonic-summing periodicity search of a [..., 'time', <freq>] cf32
    stream of spectra (see PeriodSearchBlock and the module docstring)."""
    return PeriodSearchBlock(iring, nharm, window, decim, *args, **kwargs)
