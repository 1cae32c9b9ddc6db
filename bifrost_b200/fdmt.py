"""bf.fdmt.Fdmt (mirrors python/bifrost/fdmt.py:38-76 -> bfFdmt*), plus the
sharded full-band form (extension, bfFdmtShard*)."""
import ctypes

import numpy as np

from bifrost_b200.libbifrost import _bf, _check, _get, BifrostObject
from bifrost_b200.ndarray import asarray
from bifrost_b200.Space import Space


class Fdmt(BifrostObject):
    def __init__(self):
        BifrostObject.__init__(self, _bf.bfFdmtCreate, _bf.bfFdmtDestroy)

    def init(self, nchan, max_delay, f0, df, exponent=-2.0, space='cuda'):
        space = Space(space)
        _check(_bf.bfFdmtInit(self.obj, nchan, max_delay, f0, df, exponent,
                              space.as_BFspace(), None, None))

    def execute(self, idata, odata, negative_delays=False):
        _check(_bf.bfFdmtExecute(self.obj, asarray(idata).as_BFarray(),
                                 asarray(odata).as_BFarray(), negative_delays, None, None))
        return odata

    def get_workspace_size(self, idata, odata, negative_delays=False):
        # the workspace depends on the schedule, and negative_delays takes the
        # step-by-step one: query with the flag the execute call will carry
        return _get(_bf.bfFdmtExecute, self.obj, asarray(idata).as_BFarray(),
                    asarray(odata).as_BFarray(), negative_delays, None)

    def execute_workspace(self, idata, odata, workspace_ptr, workspace_size,
                          negative_delays=False):
        size = _bf.BFsize(workspace_size)
        _check(_bf.bfFdmtExecute(self.obj, asarray(idata).as_BFarray(),
                                 asarray(odata).as_BFarray(), negative_delays,
                                 workspace_ptr, size))
        return odata

    # ---- sharded full-band transform (extension; include/bifrost_b200.h) ----
    def shard_init(self, rank, nrank):
        """This plan (initialised with the FULL band) becomes rank `rank` of
        `nrank` cooperating plans."""
        _check(_bf.bfFdmtShardInit(self.obj, rank, nrank))
        self._shard = (rank, nrank)

    def shard_workspace_size(self, idata, odata):
        size = _bf.BFsize(0)
        _check(_bf.bfFdmtShardExecute(self.obj, 0, asarray(idata).as_BFarray(), asarray(odata).as_BFarray(),
                                      None, ctypes.byref(size)))
        return int(size.value)

    def shard_execute(self, phase, idata, odata, workspace_ptr, workspace_size):
        size = _bf.BFsize(workspace_size)
        _check(_bf.bfFdmtShardExecute(self.obj, phase, asarray(idata).as_BFarray(), asarray(odata).as_BFarray(),
                                      workspace_ptr, ctypes.byref(size)))
        return odata

    def shard_execute_peers(self, idata, odata, workspace_ptr, workspace_size, peer_ptrs):
        """Phase 1 reading the split-step rows straight from every rank's
        workspace (peer_ptrs[g] = rank g's workspace as mapped here)."""
        size = _bf.BFsize(workspace_size)
        arr = (ctypes.c_void_p * len(peer_ptrs))(*[ctypes.c_void_p(int(p)) for p in peer_ptrs])
        _check(_bf.bfFdmtShardExecutePeers(self.obj, asarray(idata).as_BFarray(), asarray(odata).as_BFarray(),
                                           workspace_ptr, ctypes.byref(size), arr, len(peer_ptrs)))
        return odata

    def shard_layout(self, ntime):
        """Exchange / output layout for a gulp of `ntime` samples: dict with the
        byte offset and pitch of the split-step rows in the workspace, every
        rank's block of rows, and the (first delay, delays, owner) of every
        delay block of the last pass."""
        cap = 4096
        while True:
            info = np.zeros(cap, np.int64)
            n = ctypes.c_int(cap)
            st = _bf.bfFdmtShardQuery(self.obj, ntime, info.ctypes.data_as(ctypes.POINTER(ctypes.c_long)), ctypes.byref(n))
            if st == 0:
                break
            if cap > (1 << 22):
                _check(st)
            cap *= 8
        info = [int(v) for v in info[:n.value]]
        nrank = info[4]
        nblk = info[7 + nrank]
        tri = info[8 + nrank: 8 + nrank + 3 * nblk]
        return dict(offset=info[0], pitch=info[1], nrow=info[2], esize=info[3], nrank=nrank, split_step=info[5],
                    row_start=info[6:7 + nrank],
                    blocks=[(tri[3 * i], tri[3 * i + 1], tri[3 * i + 2]) for i in range(nblk)])
