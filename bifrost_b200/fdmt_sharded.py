"""Full-band FDMT across GPUs (extension; SURVEY 8f.1, DESIGN 6).

The reference scales FDMT by giving every GPU an independent frequency
sub-band (python/bifrost/blocks/fdmt.py:59-124 on a `gpu=` block each); the
dispersion banks of the sub-bands are then separate products.  This module
computes the FULL-BAND bank of one gulp with the channels partitioned over the
ranks of a torch.distributed group: the merge tree (src/fdmt.cu:366-387) is cut
at the step that has `world` sub-bands,

  phase 0   rank g runs the steps up to the cut on its own channels
            (bfFdmtShardExecute, no communication),
  exchange  the rows of the cut step travel between the ranks (NCCL over
            NVLink: one broadcast per rank of its block of rows, straight out
            of / into the FDMT workspace -- the only collective of the path),
  phase 1   rank g runs its share of the delay blocks of the remaining steps,

and the rows written by the ranks are, together, bit for bit the output of
bfFdmtExecute on one GPU.  One process per GPU; kernels and collectives are
ordered on the calling thread's current torch stream.

`execute(..., peer=True)` drops the exchange: the ranks map each other's
workspaces (CUDA IPC, set up once) and phase 1 stages every cut-step row with
a TMA bulk copy straight from the HBM of the GPU that produced it, over NVLink,
tile by tile while the previous tile is being merged (bfFdmtShardExecutePeers).
NCCL then only carries two barriers per gulp (phase 0 done everywhere / phase
1 done everywhere) and the optional gather.
"""
import numpy as np

from bifrost_b200.fdmt import Fdmt
from bifrost_b200 import device as _device
from bifrost_b200.ndarray import ndarray as _ndarray


class ShardedFdmt(object):
    def __init__(self, group=None):
        import torch.distributed as dist
        self._dist = dist
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.plan = Fdmt()
        self._ws = None
        self._layout = {}
        self._peer_ptrs = None
        self._peer_need = 0

    def init(self, nchan, max_delay, f0, df, exponent=-2.0):
        """Same arguments on every rank: the FULL band."""
        self.nchan, self.max_delay = nchan, max_delay
        self.plan.init(nchan, max_delay, f0, df, exponent)
        self.plan.shard_init(self.rank, self.world)
        return self

    @property
    def nchan_local(self):
        return self.nchan // self.world

    def channels(self, df_positive=True):
        """Input channels [c0, c1) of the full band that this rank holds."""
        cpr = self.nchan_local
        if df_positive:
            return self.rank * cpr, (self.rank + 1) * cpr
        return self.nchan - (self.rank + 1) * cpr, self.nchan - self.rank * cpr

    def layout(self, ntime):
        if ntime not in self._layout:
            self._layout[ntime] = self.plan.shard_layout(ntime)
        return self._layout[ntime]

    def _workspace(self, a_in, a_out):
        import torch
        need = self.plan.shard_workspace_size(a_in, a_out)
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty((need,), dtype=torch.uint8, device='cuda')
        return self._ws, need

    def exchange(self, ws, ntime):
        """Every rank's block of cut-step rows to every other rank (same byte
        offsets in every rank's workspace).  Returns the bytes this rank
        received."""
        lay = self.layout(ntime)
        got = 0
        for g in range(self.world):
            lo = lay['offset'] + lay['row_start'][g] * lay['pitch']
            hi = lay['offset'] + lay['row_start'][g + 1] * lay['pitch']
            if hi > lo:
                self._dist.broadcast(ws[lo:hi], src=self._global_rank(g), group=self.group)
                if g != self.rank:
                    got += hi - lo
        return got

    def _global_rank(self, g):
        return g if self.group is None else self._dist.get_global_rank(self.group, g)

    def map_peers(self, need):
        """Allocates this rank's peer-visible workspace (bfMalloc, i.e. its own
        cudaMalloc block) and maps every other rank's into this process (CUDA IPC;
        peer access over NVLink is enabled when a handle is opened).
        Collective; once per workspace size."""
        import ctypes
        from bifrost_b200.libbifrost import _bf, _check
        from bifrost_b200.ndarray import empty
        dist = self._dist
        self._peer_buf = empty((need,), dtype='u8', space='cuda')           # keeps the allocation alive
        mine = self._peer_buf.ctypes.data
        h = ctypes.create_string_buffer(64)
        _check(_bf.bfIpcGetHandle(mine, h))
        handles = [None] * self.world
        dist.all_gather_object(handles, bytes(h.raw), group=self.group)
        ptrs = []
        for g, hb in enumerate(handles):
            if g == self.rank:
                ptrs.append(mine)
                continue
            p = ctypes.c_void_p()
            _check(_bf.bfIpcOpenHandle(ctypes.create_string_buffer(hb, 64), ctypes.byref(p)))
            ptrs.append(p.value)
        self._peer_ptrs, self._peer_need = ptrs, need
        return ptrs

    def execute(self, x_local, out, gather_to=None, peer=False):
        """x_local: torch int8/uint8 CUDA tensor [nchan/world, ntime] (this rank's
        channels); out: torch float32 CUDA tensor [max_delay, ntime].  After
        the call `out` holds this rank's delay blocks (see layout()['blocks']);
        with gather_to=r rank r's `out` holds the whole bank.  peer=True: no
        exchange, phase 1 reads the other ranks' rows in place over NVLink."""
        import torch
        _device.set_stream(torch.cuda.current_stream().cuda_stream)
        a_in, a_out = _ndarray(base=x_local), _ndarray(base=out)
        ntime = int(x_local.shape[-1])
        if peer:
            need = self.plan.shard_workspace_size(a_in, a_out)
            if self._peer_ptrs is None or self._peer_need < need:
                self.map_peers(need)
            mine = self._peer_ptrs[self.rank]
            self.plan.shard_execute(0, a_in, a_out, mine, need)
            self._dist.barrier(group=self.group)          # every rank's rows are in its HBM
            self.plan.shard_execute_peers(a_in, a_out, mine, need, self._peer_ptrs)
            self._dist.barrier(group=self.group)          # nobody reads my workspace any more
        else:
            ws, need = self._workspace(a_in, a_out)
            self.plan.shard_execute(0, a_in, a_out, ws.data_ptr(), need)
            self.exchange(ws, ntime)
            self.plan.shard_execute(1, a_in, a_out, ws.data_ptr(), need)
        if gather_to is not None:
            self.gather(out, ntime, gather_to)
        return out

    def gather(self, out, ntime, dst):
        """Delay blocks of the other ranks into rank `dst`'s `out`."""
        dist = self._dist
        ops = []
        for d0, nd, owner in self.layout(ntime)['blocks']:
            if owner == dst:
                continue
            if self.rank == dst:
                ops.append(dist.P2POp(dist.irecv, out[d0:d0 + nd], self._global_rank(owner), self.group))
            elif self.rank == owner:
                ops.append(dist.P2POp(dist.isend, out[d0:d0 + nd], self._global_rank(dst), self.group))
        if ops:
            for r in dist.batch_isend_irecv(ops):
                r.wait()

    def owned_rows(self, ntime):
        """Boolean mask over the output delays this rank writes."""
        m = np.zeros(self.max_delay, bool)
        for d0, nd, owner in self.layout(ntime)['blocks']:
            if owner == self.rank:
                m[d0:d0 + nd] = True
        return m
