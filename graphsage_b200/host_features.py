"""A feature table kept in host memory: one GPU samples and trains from a table larger than its HBM.

The [N+1, F] rows are stored once in page-locked host memory that the device addresses directly (gs_host_register).
Only layer 0 reads the table, by the sampled ids, so every step stages the rows the batch reads into a small device
"working set"

    [C cached rows | 1 zero row | S staging rows]      (the host table's pitch and dtype, one contiguous table)

and layer 0 runs unchanged on that tensor with translated ids; layers >= 1 read row ranges of the previous output as
always.  The staging reuses the halo passes of the node-partitioned table (the working set is described to them as a
one-shard table whose `remap` is the cache map):

    gs_halo_begin -> gs_halo_claim per id list (every distinct uncached id in [0, N) takes the next staging slot)
    -> gs_host_fetch (the claimed rows over the host link) -> gs_host_translate per id list

with the count on the device, no host synchronisation and launch sizes fixed by the batch shape, so a step stays
capturable in a CUDA graph.  The hot rows (`cache_ids`, see hot_rows) are copied into the working set once and never
cross the link again.  Nothing downstream can tell where a row came from: outputs, losses and gradients are the bits the
same model computes on the table held on the device.

The sampled-block entry points (sampled_minibatch_*) stage nothing: their layer 0 reads only V_0, the sorted, unique
source ids of block 0, and needs them as fp32 rows, so gather_rows_f32 loads them in one pass (gs_host_gather_rows_f32:
cached rows from the working set's head, the rest over the link) straight into the fp32 operand.
"""
import ctypes

import numpy as np
import torch

from . import ops, parallel
from ._lib import ShardedTable, check, lib, ptr, stream_ptr


def hot_rows(adj, n_rows):
    """The `n_rows` nodes a model's batches read most, sorted int64 (possibly fewer: nodes never read are left out).
    adj: the padded adjacency table [N+1, max_degree] (numpy or tensor) - ranked by the expected reads per seed of
    parallel.expected_reads over all N seeds - or a CSR pair (indptr, indices) - ranked by in-degree."""
    if isinstance(adj, (tuple, list)):
        indptr, indices = adj
        n_nodes = len(indptr) - 1
        if n_rows <= 0:
            return np.zeros(0, dtype=np.int64)
        idx = indices if torch.is_tensor(indices) else torch.from_numpy(np.ascontiguousarray(indices))
        return parallel.top_counted(parallel.in_degrees(idx, n_nodes), min(int(n_rows), n_nodes))
    a = adj.cpu().numpy() if torch.is_tensor(adj) else np.asarray(adj)
    n_nodes = a.shape[0] - 1
    if n_rows <= 0:
        return np.zeros(0, dtype=np.int64)
    return parallel.top_scored(parallel.expected_reads(a, n_nodes, 0, n_nodes), n_rows)


def _check_cache_ids(cache_ids, n_nodes):
    if cache_ids is None:
        return np.zeros(0, dtype=np.int64)
    ids = np.asarray(cache_ids)
    if ids.ndim != 1 or (ids.size and not np.issubdtype(ids.dtype, np.integer)):
        raise ValueError("cache_ids must be a 1-D array of integer node ids")
    ids = ids.astype(np.int64)
    if ids.size and ((np.diff(ids) <= 0).any() or ids[0] < 0 or ids[-1] >= n_nodes):
        raise ValueError("cache_ids must be sorted, unique and in [0, %d)" % n_nodes)
    return ids


class HostFeatures(object):
    """A [N+1, F] float32, bfloat16 or int8 feature table in page-locked host memory, usable wherever SampleAndAggregate,
    SupervisedGraphsage and UnsupervisedGraphsage take `features`.

    table     : CPU tensor or numpy array [N+1, F]; its last row is the all-zero dummy row, as for a device table.  It is
                copied once into a host buffer of pitch ops.pad_cols(F) (16-byte rows), which is pinned and mapped.  Or an
                Int8Features table whose rows are on the CPU: its byte rows (scale included) are pinned in place, staged
                whole, and layer 0 reads the working set as an int8 table.
    cache_ids : sorted, unique int64 ids in [0, N) whose rows are copied into device memory once and served from there
                (hot_rows picks them); None caches nothing.
    device    : the GPU the working set lives on (default: the current one).

    Device memory: the working set [C + 1 + S, pitch] (C cached rows, S = the largest batch * sum(support) staged so far,
    reserved when a model is built) and two int32 [N+1] arrays (the cache map and the claim array).  close() releases
    the pinned memory."""

    def __init__(self, table, cache_ids=None, device=None):
        if isinstance(table, ops.I8Rows):            # Int8Features: rows of bytes, each holding its scale
            if table.rows.is_cuda:
                raise ValueError("HostFeatures takes a host (CPU) table; a CUDA Int8Features table is used as features "
                                 "directly")
            self.n_nodes, F = int(table.shape[0]) - 1, int(table.shape[1])
            self.dtype, self.host = torch.int8, table.rows.contiguous()
            self.pitch = self.row_bytes = self.host.shape[1]
        else:
            t = table if torch.is_tensor(table) else torch.from_numpy(np.asarray(table))
            if t.is_cuda:
                raise ValueError("HostFeatures takes a host (CPU) table; a CUDA table is used as features directly")
            if t.dim() != 2 or t.shape[0] < 1 or t.shape[1] < 1:
                raise ValueError("the table must be a 2-D [N+1, F] array with F >= 1")
            if t.dtype not in (torch.float32, torch.bfloat16):
                raise TypeError("the table must be float32 or bfloat16 (got %s)" % t.dtype)
            if bool((t[-1] != 0).any()):
                raise ValueError("the table's last row is the dummy row and must be all zero")
            self.n_nodes, F = int(t.shape[0]) - 1, int(t.shape[1])
            self.dtype = t.dtype
            self.pitch = ops.pad_cols(F)
            self.row_bytes = self.pitch * t.element_size()
            self.host = torch.zeros((self.n_nodes + 1, self.pitch), dtype=self.dtype)
            self.host[:, :F] = t
        ids = _check_cache_ids(cache_ids, self.n_nodes)
        self.shape = (self.n_nodes + 1, F)
        self.cache_ids = ids
        self.n_cached = len(ids)
        self._alias = None
        self._alias = ops.host_register(self.host)            # pinned once; every step's fetch reads through it
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        dev, C = self.device, self.n_cached
        self.cache_slot = torch.full((self.n_nodes + 1,), -1, dtype=torch.int32, device=dev)
        self.claim = torch.empty((self.n_nodes + 1,), dtype=torch.int32, device=dev)
        self.count = torch.zeros((1,), dtype=torch.int32, device=dev)
        self.ws = torch.zeros((C + 1, self.pitch), dtype=self.host.dtype, device=dev)
        self.capacity, self._captured, self._retired = 0, False, []
        if C:
            cid = torch.from_numpy(ids.astype(np.int32)).to(dev)
            self.cache_slot[cid.long()] = torch.arange(C, dtype=torch.int32, device=dev)
            ops.host_fetch(self._alias, self.row_bytes, cid, torch.full((1,), C, dtype=torch.int32, device=dev), self.ws)

    # ------------------------------------------------------------------ the working set
    def reserve(self, rows):
        """Make room for `rows` staging rows (kept across steps; the cached rows and the zero row move along)."""
        rows = int(rows)
        if rows <= self.capacity:
            return
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("HostFeatures: the working set must grow to %d staging rows inside a CUDA-graph capture; "
                               "run the batch shape once before capturing it" % rows)
        head = self.n_cached + 1
        ws = torch.empty((head + rows, self.pitch), dtype=self.ws.dtype, device=self.device)
        ws[:head].copy_(self.ws[:head])
        if self._captured:
            self._retired.append(self.ws)      # a captured graph still addresses the old buffer: keep it alive
        self.ws, self.capacity = ws, rows

    def _table(self):
        t = ShardedTable()
        t.base[0] = self.ws.data_ptr()
        t.row_start[0], t.row_start[1] = 0, self.n_nodes
        t.n_shards, t.my_shard = 1, 0
        t.n_global_rows = self.n_nodes + 1
        t.zero_row = self.n_cached
        t.remap = self.cache_slot.data_ptr()
        return t

    def stage(self, samples):
        """One step's layer-0 source: (working set [C + 1 + capacity, F] view - an ops.I8Rows over it for int8 rows -, the id
        lists translated to its rows).
        samples: the step's int32 device id lists (SampleAndAggregate.sample); all of them are read by layer 0."""
        lists = [ops._i32(s.reshape(-1), "samples") for s in samples]
        S = sum(t.numel() for t in lists)
        self.reserve(S)
        if torch.cuda.is_current_stream_capturing():
            self._captured = True
        tab = ctypes.byref(self._table())
        stage_ids = torch.empty((max(S, 1),), dtype=torch.int32, device=self.device)
        check(lib().gs_halo_begin(ptr(self.claim), self.n_nodes + 1, ptr(self.count), stream_ptr()))
        for t in lists:
            check(lib().gs_halo_claim(tab, ptr(t), t.numel(), ptr(self.claim), ptr(self.count), ptr(stage_ids), S,
                                      stream_ptr()))
        ops._launched(sum(1 for t in lists if t.numel()))
        head = self.n_cached + 1
        ops.host_fetch(self._alias, self.row_bytes, stage_ids[:S], self.count, self.ws[head:])
        out = [ops.host_translate(tab, t, self.claim, head) for t in lists]
        if self.dtype == torch.int8:
            return ops.I8Rows(self.ws, self.shape[1]), out
        return self.ws[:, :self.shape[1]], out

    def gather_rows_f32(self, ids):
        """Rows `ids` (int32 device ids) widened to fp32 in one pass (gs_host_gather_rows_f32): cached rows from the
        working set, ids outside [0, N) as the zero row, the rest over the host link - no staging, no claim.  The layer-0
        rows of a sampled block set (V_0); the fp32 [n, pad_cols(F)] buffer's [:, :F] view, the bits ops.gather_rows_f32
        gives on the same table held on the device."""
        return ops.host_gather_rows_f32(self._alias, self.ws, self.cache_slot, self.n_nodes, self.shape[1], ids)

    def close(self):
        """Unpin the host rows and drop the device buffers (the object is unusable afterwards)."""
        if getattr(self, "_alias", None) is not None:
            torch.cuda.synchronize(self.device)
            ops.host_unregister(self.host)
            self._alias = None
        self.ws = self.cache_slot = self.claim = None
        self._retired = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def step_rows(batch_size, layer_infos):
    """S of a batch: batch_size * sum(support) - every id of every layer-0 list, the most a step can stage."""
    support, total = 1, 1
    for info in reversed(layer_infos):
        support *= info.num_samples
        total += support
    return int(batch_size) * total


def stage_layer0(features, samples):
    """(src, samples) for layer 0: the working set and translated ids for a HostFeatures table, else unchanged.  The
    third value says whether src is the model's persistent table (False for a working set, rewritten every step)."""
    if isinstance(features, HostFeatures):
        src, samples = features.stage(samples)
        return src, samples, False
    return features, samples, True


def refuse_host_table(features, what):
    if isinstance(features, HostFeatures):
        raise NotImplementedError("%s with a host-memory (HostFeatures) feature table is not implemented" % what)
