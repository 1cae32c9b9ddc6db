"""bf.candidates.Candidates: friends-of-friends clustering of a peak map over
trial and time (extension, bfCandidates*; include/bifrost_b200.h).

For each leading index of peaks [..., ntrial, nblk, nfield] f32 (the output
of bfPulseSearch, nfield 3, or of bfPeriodSearch, nfield 2), the cells whose
score reaches `threshold` are grouped into clusters of friends: within
`trial_radius` trials and `pos_radius` samples of each other.
table [..., ncap, 9] f64 gets one record of RECORD_FIELDS per cluster, in
order of each cluster's first cell in time; count [..., 1] i32 gets the
number of clusters, which may exceed ncap."""
from bifrost_b200.libbifrost import _bf, _check, _exec_storage, BifrostObject
from bifrost_b200.ndarray import asarray

# The representative's (score, trial, position, field 2 or 0), then the
# cluster's member count and its trial and position extents.
RECORD_FIELDS = ['snr', 'trial', 'pos', 'width', 'members', 'trial_lo', 'trial_hi', 'pos_lo', 'pos_hi']


class Candidates(BifrostObject):
    def __init__(self):
        BifrostObject.__init__(self, _bf.bfCandidatesCreate, _bf.bfCandidatesDestroy)

    def init(self, threshold, trial_radius, pos_radius, decim):
        _check(_bf.bfCandidatesInit(self.obj, float(threshold), int(trial_radius), int(pos_radius), int(decim)))
        self.threshold, self.trial_radius = float(threshold), int(trial_radius)
        self.pos_radius, self.decim = int(pos_radius), int(decim)

    def _run(self, peaks, table, count, **storage):
        return _exec_storage(_bf.bfCandidatesExecute, self.obj, asarray(peaks).as_BFarray(),
                             asarray(table).as_BFarray(), asarray(count).as_BFarray(), **storage)

    def execute(self, peaks, table, count):
        self._run(peaks, table, count)
        return table, count

    def get_workspace_size(self, peaks, table, count):
        return self._run(peaks, table, count, query=True)

    def execute_workspace(self, peaks, table, count, workspace_ptr, workspace_size):
        self._run(peaks, table, count, workspace=(workspace_ptr, workspace_size))
        return table, count
