"""write_candidates block: friends-of-friends candidates of a pulse_search
stream, written one line per cluster to a text file (extension,
bfCandidates*; no reference counterpart)."""
import os
import warnings

import numpy as np

from bifrost_b200.pipeline import SinkBlock
from bifrost_b200.candidates import Candidates
from bifrost_b200.ndarray import zeros
from bifrost_b200.units import convert_units
from bifrost_b200.blocks import _header as H

LABELS = ['dispersion', 'time', 'peak']


def candidate_header(ihdr):
    """(decim, tsamp s, dm0, ddm pc cm^-3, widest boxcar) of a pulse_search
    output header: ['dispersion', 'time', 'peak'] f32 with time as the frame
    axis (KeyError for other labels, a missing key or leading axes such as
    beams; TypeError for another dtype)."""
    t = ihdr['_tensor']
    if list(t.get('labels') or []) != LABELS or t['shape'][1] != -1 or t['shape'][2] != 3:
        raise KeyError("Expected axes %s with time as the frame axis and 3 peak fields, got %s"
                       % (LABELS, t.get('labels')))
    H.check_dtype(t, ('f32',), 'write_candidates', 'peaks')
    decim = int(ihdr['peak_decim'])
    tsamp = convert_units(t['scales'][1][1], t['units'][1], 's') / decim
    dm0, ddm = (convert_units(v, t['units'][0], 'pc cm^-3') for v in t['scales'][0])
    return decim, tsamp, dm0, ddm, max(ihdr['boxcar_widths'])


def candidate_lines(records, sample0, tsamp, dm0, ddm):
    """One text line per record of a bfCandidates table over pulse_search
    peaks, whose first block starts at sample `sample0` of the searched
    series: snr, sample, time (s), width (samples), DM trial, DM (pc cm^-3),
    members, first sample, last sample (heimdall's column order, with the
    width in samples rather than as a filter index).  Samples and times count
    from the start of the sequence."""
    lines = []
    for r in np.asarray(records, dtype=np.float64).reshape(-1, 9):
        sample = sample0 + int(r[2])
        lines.append('%.6f\t%d\t%.9f\t%d\t%d\t%.6f\t%d\t%d\t%d\n'
                     % (r[0], sample, sample * tsamp, int(r[3]), int(r[1]), dm0 + r[1] * ddm,
                        int(r[4]), sample0 + int(r[7]), sample0 + int(r[8])))
    return lines


class CandidatesSinkBlock(SinkBlock):
    """Clusters each span of a pulse_search stream (by default one gulp of
    the search: its gulp_nframe blocks) with bfCandidates and appends the
    clusters to <path>/<name>.cand.  Clusters are found within a span, as
    pulse_search normalises within a gulp: a pulse whose above-threshold
    blocks straddle a span boundary gives one candidate in each span, each
    from its own span's blocks.  Spans with more than max_candidates clusters
    keep the first max_candidates in time order, with a warning."""

    def __init__(self, iring, path=None, threshold=6.0, trial_radius=8, pos_radius=None, max_candidates=4096,
                 *args, **kwargs):
        super(CandidatesSinkBlock, self).__init__(iring, *args, **kwargs)
        self.path = path or ''
        self.threshold, self.trial_radius = float(threshold), int(trial_radius)
        self.pos_radius = None if pos_radius is None else int(pos_radius)
        self.ncap = int(max_candidates)
        self.plan = Candidates()
        self.ofile = None

    def define_valid_input_spaces(self):
        return ('cuda',)

    def on_sequence(self, iseq):
        ihdr = iseq.header
        self.decim, self.tsamp, self.dm0, self.ddm, widest = candidate_header(ihdr)
        pos_radius = widest if self.pos_radius is None else self.pos_radius
        self.plan.init(self.threshold, self.trial_radius, pos_radius, self.decim)
        self.table = zeros((self.ncap, 9), 'f64', 'cuda')
        self.count = zeros((1,), 'i32', 'cuda')
        self.filename = os.path.join(self.path, os.path.basename(str(ihdr['name']))) + '.cand'
        self.ofile = open(self.filename, 'w')

    def on_sequence_end(self, iseq):
        if self.ofile is not None:
            self.ofile.close()
            self.ofile = None

    def on_data(self, ispan):
        self.plan.execute(ispan.data, self.table, self.count)
        n = int(np.asarray(self.count.copy('system'))[0])
        keep = min(n, self.ncap)
        if n > self.ncap:
            warnings.warn("%s: %d clusters in frames %d.., kept the first %d"
                          % (self.filename, n, ispan.frame_offset, keep))
        if keep == 0:
            return
        rows = np.asarray(self.table[:keep].copy('system'))
        self.ofile.write(''.join(candidate_lines(rows, ispan.frame_offset * self.decim,
                                                 self.tsamp, self.dm0, self.ddm)))
        self.ofile.flush()


def write_candidates(iring, path=None, threshold=6.0, trial_radius=8, pos_radius=None, max_candidates=4096,
                     *args, **kwargs):
    """Friends-of-friends candidates of a ['dispersion', 'time', 'peak']
    pulse_search stream in cuda space: peaks with S/N >= threshold within
    trial_radius DM trials and pos_radius samples (default: the widest
    boxcar) of each other form one candidate, written as one line of
    <path>/<name>.cand (see CandidatesSinkBlock and candidate_lines)."""
    return CandidatesSinkBlock(iring, path, threshold, trial_radius, pos_radius, max_candidates, *args, **kwargs)
