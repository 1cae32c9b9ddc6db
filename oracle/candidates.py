"""Friends-of-friends candidate oracle (numpy).  TEST INFRASTRUCTURE -- see
oracle/__init__.py.

The semantics of bfCandidatesExecute (include/bifrost_b200.h), restated per
leading index as members, then union-find over every friend pair, then
records:
  member: field0 >= threshold (fp64) and 0 <= field1 < decim;
  pos = fl64(j decim + field1), k = j ntrial + t;
  friends: |t - t'| <= R_t and |fl64(pos - pos')| <= R_p;
  clusters in order of their smallest k; the representative has the largest
  field0, the smaller k on ties;
  record (field0, t, pos, field2 or 0, members, t_lo, t_hi, pos_lo, pos_hi).
"""
import numpy as np

NFIELD = 9


def members(peaks, threshold, decim):
    """(t, j, pos) of the members of one [ntrial, nblk, nfield] map, in k order."""
    p = np.asarray(peaks, dtype=np.float32)
    s, o = p[..., 0].astype(np.float64), p[..., 1].astype(np.float64)
    with np.errstate(invalid='ignore'):
        m = (s >= threshold) & (o >= 0) & (o < decim)
    j, t = np.nonzero(m.T)                       # time-major: k = j ntrial + t ascending
    pos = j.astype(np.float64) * decim + o[t, j]
    return t, j, pos


def _components(n, a, b):
    """Label of each of n nodes: the smallest node of its component, for the
    edges (a[i], b[i]) (hook roots under the smaller root, then jump)."""
    parent = np.arange(n)
    while True:
        ra, rb = parent[a], parent[b]
        diff = ra != rb
        if not diff.any():
            return parent
        np.minimum.at(parent, np.maximum(ra, rb)[diff], np.minimum(ra, rb)[diff])
        while True:
            up = parent[parent]
            if np.array_equal(up, parent):
                break
            parent = up


def cluster(peaks, threshold, trial_radius, pos_radius, decim):
    """Records [nclust, 9] float64 of one [ntrial, nblk, nfield] f32 map."""
    p = np.asarray(peaks, dtype=np.float32)
    ntrial, nblk, nfield = p.shape
    t, j, pos = members(p, threshold, decim)
    n = len(t)
    if n == 0:
        return np.zeros((0, NFIELD))
    grid = np.full((ntrial, nblk), -1, np.int64)
    grid[t, j] = np.arange(n)
    a, b = [], []
    dj = pos_radius // decim + 1                 # blocks beyond this are farther than R_p
    for dt in range(0, trial_radius + 1):
        for d in range(-dj, dj + 1):
            if dt == 0 and d <= 0:
                continue                         # each pair once
            t2, j2 = t + dt, j + d
            ok = (t2 < ntrial) & (j2 >= 0) & (j2 < nblk)
            nb = np.full(n, -1, np.int64)
            nb[ok] = grid[t2[ok], j2[ok]]
            has = nb >= 0
            src, dst = np.nonzero(has)[0], nb[has]
            near = np.abs(pos[dst] - pos[src]) <= pos_radius
            a.append(src[near])
            b.append(dst[near])
    label = _components(n, np.concatenate(a), np.concatenate(b))
    roots, cid = np.unique(label, return_inverse=True)   # members are in k order: roots ascend in k
    score = p[t, j, 0]
    order = np.lexsort((np.arange(n), -score.astype(np.float64), cid))
    first = np.ones(n, bool)
    first[1:] = cid[order][1:] != cid[order][:-1]
    rep = order[first]                           # per cluster: largest score, then smallest k
    out = np.zeros((len(roots), NFIELD))
    out[:, 0] = score[rep]
    out[:, 1] = t[rep]
    out[:, 2] = pos[rep]
    if nfield == 3:
        out[:, 3] = p[t[rep], j[rep], 2]
    out[:, 4] = np.bincount(cid)
    for col, vals, red in ((5, t, np.minimum), (6, t, np.maximum), (7, pos, np.minimum), (8, pos, np.maximum)):
        acc = np.full(len(roots), np.inf if red is np.minimum else -np.inf)
        red.at(acc, cid, vals.astype(np.float64))
        out[:, col] = acc
    return out


def candidates(peaks, threshold, trial_radius, pos_radius, decim):
    """(records, count) for peaks [..., ntrial, nblk, nfield]: records is a
    list (in leading-index order) of [nclust, 9] float64 arrays and count
    the int array [..., 1] of their lengths."""
    p = np.asarray(peaks, dtype=np.float32)
    lead = p.shape[:-3]
    recs = [cluster(p[i], threshold, trial_radius, pos_radius, decim) for i in np.ndindex(*lead)]
    count = np.array([len(r) for r in recs], np.int32).reshape(lead + (1,))
    return recs, count
