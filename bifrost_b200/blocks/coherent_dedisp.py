"""coherent_dedisp block: coherent dedispersion of baseband voltages ahead of
detection (extension, bfCoherentDedisp*; no reference counterpart)."""
import math

from bifrost_b200.pipeline import TransformBlock
from bifrost_b200.coherent_dedisp import CoherentDedisp, dispersion_overlap, default_nfft
from bifrost_b200.blocks import _header as H

CD_DTYPES = ('ci4', 'ci8', 'ci16', 'cf32')
DM_UNITS = 'pc cm^-3'


def _band(ihdr):
    """(tensor, nchan, f0 MHz, df MHz) of a ['freq', ..., 'time'] voltage
    header; refuses anything the operation does not take."""
    t, nchan, f0, df, tsamp = H.channel_band(ihdr, CD_DTYPES, 'coherent_dedisp', 'voltages')
    if df == 0 or abs(abs(tsamp) * abs(df) * 1e6 - 1.0) > 1e-6:
        raise ValueError("coherent_dedisp needs critically sampled channels: |time step| (%g s) must be "
                         "1/|channel width| (%g MHz)" % (tsamp, df))
    return t, nchan, f0, df


def coherent_dedisp_header(ihdr, dm, nfft=None):
    """(output header, nfft, overlap) of coherent_dedisp(dm, nfft) on a
    ['freq', ..., 'time'] ci4 / ci8 / ci16 / cf32 sequence with header ihdr:
    the input's with dtype cf32 plus coherent_dm (and _units), coherent_nfft
    and coherent_overlap.  refdm is left alone: the delays between channels
    remain for the FDMT to search."""
    _, nchan, f0, df = _band(ihdr)
    overlap = dispersion_overlap(nchan, f0, df, dm)
    nfft = default_nfft(overlap) if nfft is None else int(nfft)
    ohdr, t = H.derive(ihdr)
    t['dtype'] = 'cf32'
    ohdr.update(coherent_dm=float(dm), coherent_dm_units=DM_UNITS, coherent_nfft=nfft,
                coherent_overlap=overlap)
    return ohdr, nfft, overlap


class CoherentDedispBlock(TransformBlock):
    """Each output frame t is the coherently dedispersed voltage of frame t,
    aligned to the arrival time at its channel's top edge.  It needs the input
    up to frame t + overlap, which the block takes as look-ahead (overlap
    frames, as the FDMT does, rounded up to whole frames of the input ring
    behind a view that merges the frame axis), so the last `overlap` (or
    rounded) frames of a sequence are never committed.  The output of each
    gulp is the operation on that gulp's span (gulp + look-ahead frames), its
    segments starting at the span's first
    frame; when gulp_nframe is a multiple of nfft - overlap, the block's output
    equals the operation on the whole stream bit for bit."""

    def __init__(self, iring, dm, nfft=None, *args, **kwargs):
        super(CoherentDedispBlock, self).__init__(iring, *args, **kwargs)
        self.dm = float(dm)
        self.nfft_arg = nfft
        self.plan = CoherentDedisp()

    def define_valid_input_spaces(self):
        return ('cuda',)

    def on_sequence(self, iseq):
        ohdr, nfft, overlap = coherent_dedisp_header(iseq.header, self.dm, self.nfft_arg)
        _, nchan, f0, df = _band(iseq.header)
        self.plan.init(nchan, f0, df, self.dm, nfft)
        self.overlap = self.plan.overlap
        return ohdr

    def define_input_overlap_nframe(self, iseq):
        # Behind a view that merges the frame axis (views.merge_axes('time',
        # 'fine_time')) the reader moves in whole frames of the ring: the
        # look-ahead is rounded up to that, which only commits fewer frames at
        # the end of the sequence.
        reader = self._readers[0]
        step = reader._den // math.gcd(reader._num, reader._den)
        return -(-self.overlap // step) * step

    def on_data(self, ispan, ospan):
        if ispan.nframe <= self.overlap:
            return 0
        self.plan.execute(ispan.data, ospan.data)


def coherent_dedisp(iring, dm, nfft=None, *args, **kwargs):
    """Coherent dedispersion of a ['freq', ..., 'time'] stream of critically
    sampled complex channels (ci4 / ci8 / ci16 / cf32, cuda space) at `dm`
    pc cm^-3 with nfft-point segments (default: default_nfft of the overlap).
    Output: cf32 (see CoherentDedispBlock and bf.coherent_dedisp)."""
    return CoherentDedispBlock(iring, dm, nfft, *args, **kwargs)
