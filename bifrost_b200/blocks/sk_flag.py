"""sk_flag block: RFI excision by windowed spectral kurtosis in front of the
FDMT (extension, bfSkFlag*; no reference counterpart)."""
from bifrost_b200.pipeline import TransformBlock
from bifrost_b200.sk_flag import SkFlag, sk_thresholds
from bifrost_b200.blocks import _header as H

SK_DTYPES = ('u8', 'u16', 'f32')


def sk_flag_header(ihdr, window, nacc=1, shape=1.0, sigma=3.0):
    """Output header of sk_flag(window, nacc, shape, sigma) on a
    [..., 'time'] u8 / u16 / f32 sequence with header ihdr: the input's,
    plus sk_window, sk_nacc, sk_shape and sk_thresholds = [lo, hi]."""
    ohdr, t = H.derive(ihdr)
    H.check_time_frames(t, SK_DTYPES, 'sk_flag', 'power')
    ohdr.update(sk_window=int(window), sk_nacc=int(nacc), sk_shape=float(shape),
                sk_thresholds=list(sk_thresholds(window, nacc, shape, sigma)))
    return ohdr


class SkFlagBlock(TransformBlock):
    """Each output frame is the input frame with flagged windows replaced by
    the row's fill.  Windows are `window` frames long and start at multiples
    of `window` in the stream (the gulp must be a multiple of it); the fill is
    the mean of the clean samples of the gulp the window belongs to, and the
    last, ragged gulp ends in a short window."""

    def __init__(self, iring, window, nacc=1, shape=1.0, sigma=3.0, *args, **kwargs):
        super(SkFlagBlock, self).__init__(iring, *args, **kwargs)
        self.window, self.nacc, self.shape, self.sigma = int(window), int(nacc), float(shape), float(sigma)
        self.plan = SkFlag()
        self.plan.init(self.window, self.nacc, self.shape, *sk_thresholds(window, nacc, shape, sigma))

    def define_valid_input_spaces(self):
        return ('cuda',)

    def on_sequence(self, iseq):
        gulp = self._gulp(iseq)
        if gulp % self.window:
            raise ValueError("gulp_nframe (%d) must be a multiple of window (%d)" % (gulp, self.window))
        ohdr = sk_flag_header(iseq.header, self.window, self.nacc, self.shape, self.sigma)
        ohdr['gulp_nframe'] = gulp
        return ohdr

    def on_data(self, ispan, ospan):
        self.plan.execute(ispan.data, ospan.data)


def sk_flag(iring, window, nacc=1, shape=1.0, sigma=3.0, *args, **kwargs):
    """Spectral-kurtosis RFI excision of a [..., 'time'] u8 / u16 / f32 power
    stream: windows of `window` samples (each the sum of `nacc` raw spectra
    with shape `shape`; 1 for power from complex voltages) whose statistic lies
    outside 1 -/+ sigma sqrt(Var) are replaced by the row's mean of clean
    samples (see SkFlagBlock and bf.sk_flag)."""
    return SkFlagBlock(iring, window, nacc, shape, sigma, *args, **kwargs)
