"""coherent_dedisp block: coherent dedispersion of baseband voltages ahead of
detection (extension, bfCoherentDedisp*; no reference counterpart).  With
detect= it is a coherent filterbank: fine channels, detection and time
integration in the same pass (bfCoherentDedispFilterbank), and only f32 power
leaves the block."""
import math

from bifrost_b200.pipeline import TransformBlock
from bifrost_b200.coherent_dedisp import CoherentDedisp, dispersion_overlap, default_nfft, NFFT_MIN
from bifrost_b200.blocks import _header as H
from bifrost_b200.blocks.detect import detect_header
from bifrost_b200.blocks.reduce import reduce_header

CD_DTYPES = ('ci4', 'ci8', 'ci16', 'cf32')
DM_UNITS = 'pc cm^-3'
DETECT_MODES = ('scalar', 'stokes', 'stokes_i', 'coherence')


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


def _check_filterbank(nfine, detect, nint):
    if detect is not None and detect not in DETECT_MODES:
        raise ValueError("detect must be None or one of %s, got %r" % (DETECT_MODES, detect))
    for name, v in (('nfine', nfine), ('nint', nint)):
        if int(v) != v or v < 1 or (detect is None and v != 1):
            raise ValueError("%s must be a positive integer, and 1 without detect; got %r" % (name, v))
    if int(nfine) & (int(nfine) - 1):
        raise ValueError("nfine must be a power of two, got %r" % (nfine,))


def coherent_filterbank_header(ihdr, dm, nfft=None, nfine=1, detect='stokes_i', nint=1):
    """(output header, nfft, overlap, mode) of coherent_dedisp(dm, nfft, nfine,
    detect, nint): the header detect(detect) -> reduce('time', nint) would give
    coherent_dedisp's output, with the freq axis split into nchan nfine fine
    channels (scales [f0 - df/2 + df'/2, df'], df' = df / nfine), the time step
    multiplied by nfine (and nint), and coherent_nfine.  mode is the detection
    the operation runs ('scalar' when there is no 2-long pol axis)."""
    _check_filterbank(nfine, detect, nint)
    ohdr, nfft, overlap = coherent_dedisp_header(ihdr, dm, nfft)
    nfine, nint = int(nfine), int(nint)
    if nfft // nfine < NFFT_MIN:
        raise ValueError("nfft / nfine = %d / %d is below %d" % (nfft, nfine, NFFT_MIN))
    if nfine * nint > nfft - overlap:
        raise ValueError("nfine x nint = %d exceeds nfft - overlap = %d" % (nfine * nint, nfft - overlap))
    if len(ohdr['_tensor']['shape']) not in (2, 3):
        raise ValueError("a coherent filterbank takes ['freq', 'time'] or ['freq', <pol>, 'time'] voltages, got %s"
                         % (ohdr['_tensor'].get('labels'),))
    ohdr, _, npol = detect_header(ohdr, detect)
    mode = detect if npol == 2 else 'scalar'
    if nint > 1:
        ohdr = reduce_header(ohdr, 'time', nint, 'sum')[0]
    t = ohdr['_tensor']
    t['shape'][0] *= nfine
    if t.get('scales') and t['scales'][0] is not None:
        f0, df = t['scales'][0]
        dff = df / nfine
        t['scales'][0] = [f0 - 0.5 * df + 0.5 * dff, dff]
    H.scale_step(t, len(t['shape']) - 1, nfine)
    gulp = ihdr.get('gulp_nframe')
    if gulp:
        ohdr['gulp_nframe'] = max(int(gulp) // (nfine * nint), 1)
    ohdr['coherent_nfine'] = nfine
    return ohdr, nfft, overlap, mode


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
    equals the operation on the whole stream bit for bit.

    With detect= the block runs the coherent filterbank
    (CoherentDedisp.filterbank): each output frame is the sum of nint detected
    fine samples of nfine fine channels per channel.  The gulp must then be a
    multiple of nfine nint, and the look-ahead is also rounded up to one; when
    the gulp is a multiple of the filterbank's segment step
    nfine nint floor((nfft - overlap) / (nfine nint)), the output equals the
    operation on the whole stream bit for bit."""

    def __init__(self, iring, dm, nfft=None, nfine=1, detect=None, nint=1, *args, **kwargs):
        _check_filterbank(nfine, detect, nint)
        super(CoherentDedispBlock, self).__init__(iring, *args, **kwargs)
        self.dm = float(dm)
        self.nfft_arg = nfft
        self.nfine, self.detect, self.nint = int(nfine), detect, int(nint)
        self.q = self.nfine * self.nint if detect is not None else 1
        self.plan = CoherentDedisp()

    def define_valid_input_spaces(self):
        return ('cuda',)

    def define_output_nframes(self, input_nframe):
        return input_nframe // self.q

    def on_sequence(self, iseq):
        if self.detect is None:
            ohdr, nfft, overlap = coherent_dedisp_header(iseq.header, self.dm, self.nfft_arg)
        else:
            ohdr, nfft, overlap, self.mode = coherent_filterbank_header(
                iseq.header, self.dm, self.nfft_arg, self.nfine, self.detect, self.nint)
            gulp = self._gulp(iseq)
            if gulp % self.q:
                raise ValueError("gulp_nframe (%i) is not a multiple of nfine x nint (%i)" % (gulp, self.q))
        _, nchan, f0, df = _band(iseq.header)
        self.plan.init(nchan, f0, df, self.dm, nfft)
        self.overlap = self.plan.overlap
        return ohdr

    def define_input_overlap_nframe(self, iseq):
        # Behind a view that merges the frame axis (views.merge_axes('time',
        # 'fine_time')) the reader moves in whole frames of the ring: the
        # look-ahead is rounded up to that, which only commits fewer frames at
        # the end of the sequence.  The filterbank takes whole outputs only.
        reader = self._readers[0]
        step = reader._den // math.gcd(reader._num, reader._den)
        step = step * self.q // math.gcd(step, self.q)
        return -(-self.overlap // step) * step

    def on_data(self, ispan, ospan):
        if ispan.nframe <= self.overlap:
            return 0
        if self.detect is None:
            self.plan.execute(ispan.data, ospan.data)
            return
        nout = ispan.nframe // self.q
        idata = ispan.data
        odata = ospan.data
        if len(idata.shape) == 2:
            idata = idata.reshape(idata.shape[0], 1, idata.shape[1])
            odata = odata.reshape(odata.shape[0], 1, odata.shape[1])
        self.plan.filterbank(idata[:, :, :nout * self.q], odata[:, :, :nout], self.nfine, self.mode, self.nint)


def coherent_dedisp(iring, dm, nfft=None, nfine=1, detect=None, nint=1, *args, **kwargs):
    """Coherent dedispersion of a ['freq', ..., 'time'] stream of critically
    sampled complex channels (ci4 / ci8 / ci16 / cf32, cuda space) at `dm`
    pc cm^-3 with nfft-point segments (default: default_nfft of the overlap).
    Output: cf32 (see CoherentDedispBlock and bf.coherent_dedisp).

    detect='scalar' | 'stokes' | 'stokes_i' | 'coherence' makes it a coherent
    filterbank: f32 power of nfine fine channels per channel (a power of two,
    nfft / nfine >= 256), each aligned to its own top edge and summed over
    nint samples, from ['freq', 'time'] or ['freq', <pol>, 'time'] voltages
    (see coherent_filterbank_header).  nfine and nint need detect."""
    return CoherentDedispBlock(iring, dm, nfft, nfine, detect, nint, *args, **kwargs)
