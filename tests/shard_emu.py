"""A node-partitioned feature table with every shard in this one GPU's memory.

`EmulatedShards` stands in for `graphsage_b200.parallel.ShardedFeatures` wherever ops.py and models.py read one: it has
the same attributes and fills a `_lib.ShardedTable` by hand, with one separate device allocation per shard instead of a
CUDA IPC mapping of another GPU's buffer.  The sharded kernels only need each `base[r]` to be a 16-byte-aligned device
pointer, so every code path of a multi-GPU table (owner search, replicas, locators, halo staging) runs on one GPU.

Layout (the one ShardedFeatures documents): shard r's buffer holds the rows of the global nodes
[row_start[r], row_start[r+1]); my shard's buffer continues with the zero row and then the replica rows.  Whatever a
correct kernel never reads is poisoned with NaN, so an addressing or masking error shows up as a wrong value or a NaN:
  - columns F .. pitch-1 of every row (the zero row's first F columns stay 0);
  - one guard row at the end of every buffer (it also keeps an off-by-one read inside the allocation).
"""
import ctypes

import numpy as np
import torch

from graphsage_b200 import _lib
from graphsage_b200.ops import pad_cols


class EmulatedShards(object):
    """dense: float32 [N, F] (the N real rows, no dummy row); row_start: the partition bounds (n_shards + 1 entries from 0
    to N); my_shard: the shard playing "this GPU"; replica_ids: optional sorted unique remote ids held by my shard."""

    def __init__(self, dense, row_start, my_shard, replica_ids=None, stage_halo=False, device="cuda"):
        dense = np.ascontiguousarray(dense, dtype=np.float32)
        N, F = dense.shape
        self.row_start = [int(x) for x in row_start]
        self.world, self.rank = len(self.row_start) - 1, int(my_shard)
        if self.row_start[0] != 0 or self.row_start[-1] != N or not 0 <= self.rank < self.world:
            raise ValueError("row_start must run from 0 to N and my_shard must name one of its shards")
        self.n_nodes = N
        self.shape = (N + 1, F)
        self.pitch = pad_cols(F)
        self.device = torch.device(device)
        self.stage_halo = bool(stage_halo)
        lo, hi = self.row_start[self.rank], self.row_start[self.rank + 1]
        self.lo, self.hi, self.n_local = lo, hi, hi - lo
        rep = np.zeros(0, np.int64) if replica_ids is None else np.asarray(replica_ids, dtype=np.int64).reshape(-1)
        if len(rep) and ((np.diff(rep) <= 0).any() or rep[0] < 0 or rep[-1] >= N or ((rep >= lo) & (rep < hi)).any()):
            raise ValueError("replica_ids must be sorted, unique, in range and not owned by my shard")
        self.replica_ids = rep
        self.zero_row = self.n_local
        self.buffers = []
        for r in range(self.world):
            a, b = self.row_start[r], self.row_start[r + 1]
            rows = dense[a:b]
            if r == self.rank:
                rows = np.vstack([rows, np.zeros((1, F), np.float32), dense[rep]])
            buf = np.full((len(rows) + 1, self.pitch), np.nan, np.float32)     # + the NaN guard row
            buf[:len(rows), :F] = rows
            self.buffers.append(torch.from_numpy(buf).to(self.device))
        self.local = self.buffers[self.rank]
        self.remap = None
        if len(rep):                                 # exactly as ShardedFeatures.__init__ builds it
            rid = torch.from_numpy(rep).to(self.device)
            remap = torch.full((N + 1,), -1, dtype=torch.int32, device=self.device)
            remap[lo:hi] = torch.arange(self.n_local, dtype=torch.int32, device=self.device)
            remap[N] = self.n_local
            remap[rid] = self.n_local + 1 + torch.arange(len(rep), dtype=torch.int32, device=self.device)
            self.remap = remap
        self._table = _lib.ShardedTable()
        for r, buf in enumerate(self.buffers):
            self._table.base[r] = buf.data_ptr()
        for r in range(self.world + 1):
            self._table.row_start[r] = self.row_start[r]
        self._table.n_shards = self.world
        self._table.my_shard = self.rank
        self._table.n_global_rows = N + 1
        self._table.zero_row = self.zero_row
        self._table.remap = 0 if self.remap is None else self.remap.data_ptr()

    def c_table(self):
        return ctypes.byref(self._table)

    def table_copy(self):
        """A copy of the C table, to be altered by a test without touching this emulator's."""
        t = _lib.ShardedTable()
        ctypes.memmove(ctypes.byref(t), ctypes.byref(self._table), ctypes.sizeof(t))
        return t

    def replica_rows(self):
        """The replica rows of my shard's buffer ([n_replicas, F] view)."""
        a = self.n_local + 1
        return self.local[a:a + len(self.replica_ids), :self.shape[1]]

    def close(self):
        torch.cuda.synchronize()
        self.buffers, self.local, self.remap = [], None, None
