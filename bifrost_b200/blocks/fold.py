"""fold block: phase-binned pulsar profiles of a power stream, one per
subintegration (extension, bfFold*; no reference counterpart)."""
import numpy as np

from bifrost_b200.pipeline import TransformBlock
from bifrost_b200.fold import Fold, dispersion_delays
from bifrost_b200.map import map as bf_map
from bifrost_b200.ndarray import empty
from bifrost_b200.units import convert_units
from bifrost_b200.blocks import _header as H

FOLD_DTYPES = ('u8', 'u16', 'f32')
MJD_UNIX_EPOCH = 40587
COUNT_MAX = 1 << 31


def fold_header(ihdr, nbin, nu, nudot=0., nuddot=0., pepoch=None, dm=None, tsubint=None, gulp_nframe=None):
    """(output header, delays s, tsamp s, t0 s, nsamp_sub) of fold(nbin, nu,
    nudot, nuddot, pepoch, dm, tsubint) on a ['freq', ..., 'time'] u8 / u16 /
    f32 sequence with header ihdr, read gulp_nframe frames at a time (default:
    the header's gulp_nframe).

    Channel reference frequencies are the top edges f_c + |df|/2 after
    coherent dedispersion (the header has coherent_dm), else the centres f_c;
    fref is the highest of them, so every delay is >= 0.  dm=None takes
    coherent_dm.  pepoch=None puts phase 0 at the sequence's first sample,
    otherwise it is the ephemeris epoch as an MJD and t0 = time origin (unix
    s) - (pepoch - 40587) 86400.  A subintegration is tsubint s rounded to
    whole samples, which must be a positive multiple of the gulp (None: one
    gulp)."""
    t, nchan, f0, df, tsamp = H.channel_band(ihdr, FOLD_DTYPES, 'fold', 'power')
    tsamp = abs(tsamp)
    if tsamp == 0:
        raise ValueError("the time axis has no sampling step")
    if dm is None:
        if 'coherent_dm' not in ihdr:
            raise ValueError("fold needs dm= when the input was not coherently dedispersed")
        dm = ihdr['coherent_dm']
    dm = float(dm)
    freqs = f0 + df * np.arange(nchan, dtype=np.float64)
    if 'coherent_dm' in ihdr:
        freqs = freqs + 0.5 * abs(df)
    fref = float(freqs.max())
    delays = dispersion_delays(freqs, dm, fref)
    origin = convert_units(t['scales'][-1][0], t['units'][-1], 's')
    t0 = 0.0 if pepoch is None else origin - (float(pepoch) - MJD_UNIX_EPOCH) * 86400.0
    gulp = int(gulp_nframe if gulp_nframe is not None else ihdr.get('gulp_nframe') or 1)
    if tsubint is None:
        nsamp_sub = gulp
    else:
        nsamp_sub = int(round(float(tsubint) / tsamp))
        if nsamp_sub <= 0 or nsamp_sub % gulp:
            raise ValueError("tsubint = %g s is %d samples: not a positive multiple of the gulp (%d)"
                             % (tsubint, nsamp_sub, gulp))
    if nsamp_sub >= COUNT_MAX:
        raise ValueError("a subintegration of %d samples overflows the 32-bit counts" % nsamp_sub)

    ohdr, o = H.derive(ihdr)
    nd = len(t['shape'])
    picks = [nd - 1] + list(range(nd - 1))          # time first, then freq and the axes between
    H.remap_axes(t, o, picks)
    o['shape'] = [-1] + list(t['shape'][:-1]) + [int(nbin)]
    o['dtype'] = 'f32'
    if 'labels' in o:
        o['labels'] = ['time'] + list(t['labels'][:-1]) + ['phase']
    if 'scales' in o:
        tstart, tstep = t['scales'][-1]
        o['scales'] = [[tstart, abs(tstep) * nsamp_sub]] + o['scales'][1:] + [[0.0, 1.0 / int(nbin)]]
    if 'units' in o:
        o['units'] = o['units'] + [None]
    ohdr.update(fold_nbin=int(nbin), fold_nu=float(nu), fold_nudot=float(nudot), fold_nuddot=float(nuddot),
                fold_pepoch=None if pepoch is None else float(pepoch), fold_dm=dm, fold_fref=fref,
                fold_nsamp_sub=nsamp_sub)
    ohdr['gulp_nframe'] = 1
    return ohdr, delays, tsamp, t0, nsamp_sub


class FoldBlock(TransformBlock):
    """Each output frame is one subintegration of nsamp_sub input frames: per
    row and phase bin, the mean of the samples folded into it (0 for a bin no
    sample fell into).  Sums and counts are kept in fp64-added f32 / i32
    buffers of the block (bfFoldExecute with accumulate); a partial last
    subintegration is not emitted."""

    def __init__(self, iring, nbin, nu, nudot=0., nuddot=0., pepoch=None, dm=None, tsubint=None,
                 *args, **kwargs):
        super(FoldBlock, self).__init__(iring, *args, **kwargs)
        self.nbin, self.nu, self.nudot, self.nuddot = int(nbin), float(nu), float(nudot), float(nuddot)
        self.pepoch, self.dm, self.tsubint = pepoch, dm, tsubint
        self.plan = Fold()

    def define_valid_input_spaces(self):
        return ('cuda',)

    def define_output_nframes(self, input_nframe):
        return 1

    def on_sequence(self, iseq):
        ohdr, delays, tsamp, t0, self.nsamp_sub = fold_header(
            iseq.header, self.nbin, self.nu, self.nudot, self.nuddot, self.pepoch, self.dm, self.tsubint,
            self._gulp(iseq))
        self.plan.init(self.nbin, delays, tsamp, t0, self.nu, self.nudot, self.nuddot)
        shape = list(ohdr['_tensor']['shape'][1:])
        self.sums = empty(shape, dtype='f32', space='cuda')
        self.counts = empty([shape[0], self.nbin], dtype='i32', space='cuda')
        self.nframe_done = 0
        return ohdr

    def on_data(self, ispan, ospan):
        self.plan.execute(ispan.data, self.sums, self.counts, first=ispan.frame_offset,
                          accumulate=self.nframe_done > 0)
        self.nframe_done += ispan.nframe
        if self.nframe_done < self.nsamp_sub:
            return 0
        self.nframe_done = 0
        nchan = self.sums.shape[0]
        rows = int(np.prod(self.sums.shape[1:-1], dtype=np.int64))
        shape = (nchan, rows, self.nbin)
        bf_map("y(c,r,b) = n(c,b) ? s(c,r,b) / (float)n(c,b) : 0.f",
               {'y': ospan.data.reshape(shape), 's': self.sums.reshape(shape), 'n': self.counts},
               axis_names=('c', 'r', 'b'), shape=shape)
        return 1


def fold(iring, nbin, nu, nudot=0., nuddot=0., pepoch=None, dm=None, tsubint=None, *args, **kwargs):
    """Fold a ['freq', ..., 'time'] u8 / u16 / f32 power stream (cuda space)
    at spin frequency nu Hz (nudot Hz/s, nuddot Hz/s^2, epoch pepoch MJD) into
    nbin phase bins, dedispersing at dm (default: the header's coherent_dm)
    and emitting one mean profile per tsubint seconds (default: per gulp).
    Output: f32 ['time', 'freq', ..., 'phase'] (see FoldBlock, fold_header and
    bf.fold)."""
    return FoldBlock(iring, nbin, nu, nudot, nuddot, pepoch, dm, tsubint, *args, **kwargs)
