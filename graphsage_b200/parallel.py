"""Multi-GPU: node-partitioned feature table with the halo exchange fused into the gather.

One process per GPU (torch.distributed for bootstrap, seed routing, barriers and the training step's one gradient
all-reduce).  Rank r owns the feature rows of the global nodes [row_start[r], row_start[r+1]) - equal ranges
(`uniform_bounds`) or cuts moved to community starts (`community_bounds`); every rank maps every shard through CUDA IPC
(NVLink / NVSwitch peer memory), and the gather kernels (gs_gather_mean_sharded / gs_gather_rows_sharded) resolve
each id to `base[owner] + (id - row_start[owner]) * pitch`: remote rows are pulled by the
consuming kernel's own bulk copies, so no collective sits on the data path.  A rank may also keep replicas of the
remote rows its batches read most (`hot_remote_rows`, `hot_remote_rows_csr`) behind its own rows; ids are then resolved
once per step to locators (ops.translate_ids) and replica hits are local reads.  GS_HALO_STAGING=1 switches to the
claim / fetch / translate staging pass (every remote row of a step crosses NVLink once; measured slower at 2 GPUs, so
opt-in).  The reference is single-device (supervised_train.py:59); this is new design (SURVEY 8e).

Seeds are routed to their owner (`route_seeds`, owner-computes), so hop-0 self rows are always local; how many of the
hop-1 / hop-2 rows are remote is decided by the partition (relabel nodes by community first: `locality_order`) and by
the replica budget (`default_cache_rows`).  Data-parallel training: `broadcast_parameters` + `allreduce_gradients`.
"""
import ctypes
import os

import numpy as np
import torch

from . import _lib
from ._lib import ShardedTable, check, lib
from .ops import pad_cols


def rows_per_shard(n_nodes, world):
    return (int(n_nodes) + world - 1) // world


def uniform_bounds(n_nodes, world):
    """row_start of the equal-range partition: shard r owns [r*R, min(N, (r+1)*R)), R = ceil(N / world)."""
    R = rows_per_shard(n_nodes, world)
    return [min(int(n_nodes), r * R) for r in range(world)] + [int(n_nodes)]


def community_bounds(comm, world):
    """row_start aligned with communities: `comm` is the community of every node with communities CONTIGUOUS in id
    order (synthetic.reddit_like relabels nodes that way); each cut is moved to the nearest community start, so no
    community straddles two GPUs (SURVEY 8e (i): locality-aware partition)."""
    comm = np.asarray(comm)
    n = len(comm)
    starts = np.concatenate([[0], np.nonzero(comm[1:] != comm[:-1])[0] + 1, [n]])
    bounds = [0]
    for r in range(1, world):
        c = int(starts[np.argmin(np.abs(starts - r * n / float(world)))])
        bounds.append(max(c, bounds[-1]))
    return bounds + [n]


def owner_of(ids, n_nodes, world, row_start=None):
    """Owner rank of each global id (numpy or torch); ids outside [0, n_nodes) - the dummy id included - map to -1
    (every rank has a zero row)."""
    rs = uniform_bounds(n_nodes, world) if row_start is None else list(row_start)
    if torch.is_tensor(ids):
        b = torch.as_tensor(rs[1:-1], dtype=ids.dtype, device=ids.device)
        o = torch.bucketize(ids, b, right=True)
        return torch.where((ids < 0) | (ids >= n_nodes), torch.full_like(o, -1), o)
    o = np.searchsorted(np.asarray(rs[1:-1]), ids, side="right")
    return np.where((ids < 0) | (ids >= n_nodes), -1, o)


def default_cache_rows(n_nodes, world):
    """Replica budget used by bench.py when none is given: a quarter of the table per GPU, whatever the GPU count
    (at 8 GPUs a GPU then holds its own eighth plus twice as many replica rows: 3/8 of the table)."""
    return (int(n_nodes) + 3) // 4 if world > 1 else 0


def expected_reads(adj, n_nodes, lo, hi):
    """Expected reads of every node [n_nodes] per seed drawn from [lo, hi), by the access probabilities the padded table
    implies: hop-1 nodes are the entries of the seeds' adjacency rows, hop-2 nodes the entries of THEIR rows; a node's
    score is hop 1 + hop 2, fanout-weighted 10 and 250.  float64."""
    adj = np.asarray(adj)
    md = adj.shape[1]
    p1 = np.bincount(adj[lo:hi].reshape(-1), minlength=n_nodes + 1).astype(np.float64)
    p1 /= max(p1.sum(), 1.0)                                  # P(a hop-1 draw lands on u)
    nz = np.nonzero(p1[:n_nodes])[0]
    p2 = np.bincount(adj[nz].reshape(-1), weights=np.repeat(p1[nz] / md, md), minlength=n_nodes + 1)
    return (10.0 * p1 + 250.0 * p2)[:n_nodes]


def top_scored(score, n_rows):
    """The (at most) n_rows ids of highest positive score, sorted int64."""
    n_rows = int(min(n_rows, int((score > 0).sum())))
    if n_rows <= 0:
        return np.zeros(0, dtype=np.int64)
    hot = np.argpartition(-score, n_rows - 1)[:n_rows]
    return np.sort(hot).astype(np.int64)


def hot_remote_rows(adj, n_nodes, world, rank, n_rows, row_start=None):
    """The `n_rows` REMOTE nodes this rank's batches will read most, by the access probabilities the padded table
    implies for seeds owned by `rank` (owner-computes): expected_reads over the own rows.  Returns sorted int64 ids
    (possibly fewer than n_rows)."""
    if n_rows <= 0 or world <= 1:
        return np.zeros(0, dtype=np.int64)
    rs = uniform_bounds(n_nodes, world) if row_start is None else list(row_start)
    lo, hi = rs[rank], rs[rank + 1]
    score = expected_reads(adj, n_nodes, lo, hi)
    score[lo:hi] = -1.0                                       # own rows need no replica
    return top_scored(score, n_rows)


def locality_order(comm):
    """Permutation `order` (new id -> old id) that makes communities contiguous, so that contiguous
    equal ranges align with communities; returns (order, inverse) with inverse[old] = new."""
    order = np.argsort(comm, kind="stable")
    inv = np.empty_like(order)
    inv[order] = np.arange(len(order))
    return order, inv


def relabel_graph(indptr, indices, order, inv):
    """CSR of the graph with node ids renamed old -> inv[old] (rows reordered accordingly)."""
    indptr = np.asarray(indptr)
    deg = np.diff(indptr)[order]
    new_ptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    src_start = indptr[:-1][order]
    ent = np.arange(new_ptr[-1]) - np.repeat(new_ptr[:-1], deg) + np.repeat(src_start, deg)
    return new_ptr, inv[np.asarray(indices)[ent]].astype(np.int32)


def route_seeds(seeds, n_nodes, group=None, row_start=None):
    """Owner-computes routing: every rank passes the seeds it was handed; returns the seeds this rank owns
    (all_to_all of variable-length id lists; works on gloo and nccl)."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    seeds = seeds.reshape(-1)
    own = owner_of(seeds, n_nodes, world, row_start).clamp(min=0)
    order = torch.argsort(own, stable=True)
    send = seeds[order].contiguous()
    counts = torch.bincount(own, minlength=world)
    recv_counts = torch.empty_like(counts)
    dist.all_to_all_single(recv_counts, counts, group=group)
    out = torch.empty(int(recv_counts.sum().item()), dtype=seeds.dtype, device=seeds.device)
    dist.all_to_all_single(out, send, output_split_sizes=recv_counts.tolist(), input_split_sizes=counts.tolist(),
                           group=group)
    return out


def in_degrees(indices, n_nodes, chunk=1 << 27):
    """How many adjacency lists hold each node (int64 [n_nodes] on indices' device), counted in chunks of the CSR column
    array; under uniform neighbour sampling a node is read in proportion to it."""
    cnt = torch.zeros((n_nodes,), dtype=torch.int64, device=indices.device)
    for i in range(0, indices.numel(), chunk):
        part = indices[i:i + chunk].long()
        cnt += torch.bincount(part.clamp_(0, n_nodes - 1), minlength=n_nodes)
        del part
    return cnt


def top_counted(cnt, n_rows):
    """The (at most) n_rows ids of highest positive count (cnt: int64 tensor), sorted int64 on the host."""
    hot = torch.topk(cnt, int(n_rows), sorted=False).indices
    hot = hot[cnt[hot] > 0]
    return np.sort(hot.cpu().numpy()).astype(np.int64)


def hot_remote_rows_csr(indices, n_nodes, world, rank, n_rows, row_start=None, chunk=1 << 27):
    """Replica choice for a graph held as CSR on the device (no padded table): the `n_rows` remote nodes with the highest
    in-degree (in_degrees).  `indices` is the CSR column array (CUDA int32); returns sorted int64 ids on the host."""
    if n_rows <= 0 or world <= 1:
        return np.zeros(0, dtype=np.int64)
    rs = uniform_bounds(n_nodes, world) if row_start is None else list(row_start)
    lo, hi = rs[rank], rs[rank + 1]
    cnt = in_degrees(indices, n_nodes, chunk)
    cnt[lo:hi] = -1
    return top_counted(cnt, min(n_rows, n_nodes - (hi - lo)))


def broadcast_parameters(params, src=0, group=None):
    """Make every rank start from rank `src`'s weights (data-parallel training: the aggregator / head weights are
    replicated, < 1 MB in total)."""
    import torch.distributed as dist
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    with torch.no_grad():
        for p in params:
            dist.broadcast(p.data, src=src, group=group)


def allreduce_gradients(params, group=None):
    """The ONE collective of the data-parallel training step (SURVEY 8e: "one gradient all-reduce of < 1 MB"): the
    gradients of all replicated weights are packed into a single buffer, summed over the ranks (NCCL all-reduce over
    NVLink / gloo on CPU), divided by the world size - the mean over the global batch, since every rank's loss is a
    mean over its own equally sized batch - and written back.  Parameters without a gradient contribute zeros so that
    the buffer has the same layout on every rank.  Returns the number of bytes reduced."""
    import torch.distributed as dist
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return 0
    params = list(params)
    if not params:
        return 0
    world = dist.get_world_size(group)
    flat = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1).to(torch.float32) for p in params])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    flat.div_(float(world))
    off = 0
    for p in params:
        n = p.numel()
        g = flat[off:off + n].view_as(p).to(p.dtype)
        if p.grad is None:
            p.grad = g.clone()
        else:
            p.grad.copy_(g)
        off += n
    return flat.numel() * 4


class _CudaView(object):
    """Expose a raw device pointer to torch through __cuda_array_interface__ (no copy)."""

    def __init__(self, ptr, shape, typestr="<f4"):
        self.__cuda_array_interface__ = {"data": (int(ptr), False), "shape": tuple(shape), "typestr": typestr,
                                         "version": 3, "strides": None}


class ShardedFeatures(object):
    """This rank's shard of a node-partitioned [N+1, F] fp32 feature table plus peer mappings of all others.

    local_rows : float32 [n_local, F] rows of the global nodes [row_start[rank], row_start[rank+1]) (numpy or tensor).
    row_start  : partition bounds (len world + 1); default = equal ranges (uniform_bounds).
    replica_ids / replica_rows : optional remote node ids (sorted, unique, none owned by this rank) and their feature
        rows [len(replica_ids), F]: kept in this rank's own buffer and served locally (hot-row replication, SURVEY 8e iii).
    The local buffer is [n_local + 1 + n_replicas, pitch]: own rows, the zero row (the dummy row, reference
    supervised_train.py:133-135, local on every rank), then the replicas.
    """

    def __init__(self, local_rows, n_nodes, group=None, device=None, row_start=None, replica_ids=None, replica_rows=None,
                 n_features=None):
        import torch.distributed as dist
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.n_nodes = int(n_nodes)
        self.row_start = [int(x) for x in (uniform_bounds(n_nodes, self.world) if row_start is None else row_start)]
        if len(self.row_start) != self.world + 1 or self.row_start[0] != 0 or self.row_start[-1] != self.n_nodes:
            raise ValueError("row_start must have world + 1 entries running from 0 to n_nodes")
        if self.world > _lib.MAX_SHARDS:
            raise ValueError("at most %d shards" % _lib.MAX_SHARDS)
        lo, hi = self.row_start[self.rank], self.row_start[self.rank + 1]
        n_local = hi - lo
        self.lo, self.hi, self.n_local = lo, hi, n_local
        if local_rows is None:
            # big shards are produced on the device: the caller fills self.local[:n_local, :F] itself (then fill_replicas())
            if not n_features:
                raise ValueError("n_features is required when local_rows is None")
            F = int(n_features)
        else:
            local_rows = torch.as_tensor(local_rows, dtype=torch.float32)
            F = local_rows.shape[1]
            if local_rows.shape[0] != n_local:
                raise ValueError("rank %d must pass %d rows (got %d)" % (self.rank, n_local, local_rows.shape[0]))
        rep_ids = np.zeros(0, np.int64) if replica_ids is None else np.asarray(replica_ids, dtype=np.int64).reshape(-1)
        if len(rep_ids):
            if replica_rows is not None and len(replica_rows) != len(rep_ids):
                raise ValueError("replica_rows must hold one row per replica id")
            if (np.diff(rep_ids) <= 0).any() or rep_ids[0] < 0 or rep_ids[-1] >= self.n_nodes \
                    or ((rep_ids >= lo) & (rep_ids < hi)).any():
                raise ValueError("replica_ids must be sorted, unique, in range and not owned by this rank")
        self.replica_ids = rep_ids
        self.shape = (self.n_nodes + 1, F)
        self.stage_halo = os.environ.get("GS_HALO_STAGING", "0") == "1"   # opt-in: fetch every remote row of a step once (ops._gather_mean_sharded); measured slower at 2 GPUs
        self.pitch = pad_cols(F)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        rows_total = n_local + 1 + len(rep_ids)
        nbytes = rows_total * self.pitch * 4
        p = ctypes.c_void_p()
        check(lib().gs_shard_alloc(nbytes, ctypes.byref(p)))
        self._own_ptr = p.value
        self.local = torch.as_tensor(_CudaView(p.value, (rows_total, self.pitch)), device=self.device)
        self.local.zero_()
        if local_rows is not None:
            self.local[:n_local, :F] = local_rows.to(self.device)
        self.zero_row = n_local
        self.remap, self._pending_remap = None, None
        if len(rep_ids):
            rid = torch.from_numpy(rep_ids).to(self.device)
            remap = torch.full((self.n_nodes + 1,), -1, dtype=torch.int32, device=self.device)
            remap[lo:hi] = torch.arange(n_local, dtype=torch.int32, device=self.device)
            remap[self.n_nodes] = n_local
            remap[rid] = n_local + 1 + torch.arange(len(rep_ids), dtype=torch.int32, device=self.device)
            if replica_rows is not None:
                self.local[n_local + 1:, :F] = torch.as_tensor(replica_rows, dtype=torch.float32).to(self.device)
                self.remap = remap
            else:
                self._pending_remap = remap                  # installed by fill_replicas() once the owners' rows exist
        torch.cuda.synchronize()
        # exchange IPC handles
        handle = ctypes.create_string_buffer(64)
        check(lib().gs_ipc_export(p, handle))
        handles = [None] * self.world
        if self.world > 1:
            dist.all_gather_object(handles, bytes(handle.raw), group=group)
        else:
            handles[0] = bytes(handle.raw)
        self._peer_ptrs = []
        self._table = ShardedTable()
        for r in range(self.world):
            if r == self.rank:
                self._table.base[r] = p.value
            else:
                q = ctypes.c_void_p()
                check(lib().gs_ipc_import(handles[r], ctypes.byref(q)))
                self._peer_ptrs.append(q.value)
                self._table.base[r] = q.value
        for r in range(self.world + 1):
            self._table.row_start[r] = self.row_start[r]
        self._table.n_shards = self.world
        self._table.my_shard = self.rank
        self._table.n_global_rows = self.n_nodes + 1
        self._table.zero_row = self.zero_row
        self._table.remap = 0 if self.remap is None else self.remap.data_ptr()
        if self.world > 1:
            dist.barrier(group=group)

    def c_table(self):
        return ctypes.byref(self._table)

    def fill_replicas(self, chunk=1 << 20):
        """Copy the replica rows from their owners (peer loads over NVLink) after EVERY rank has filled its own rows;
        collective (barriers).  Only needed when the shard was built with replica_ids but without replica_rows."""
        import torch.distributed as dist
        from . import ops
        torch.cuda.synchronize()
        if self.world > 1 and dist.is_initialized():
            dist.barrier(group=self.group)                    # every owner's rows are in place
        if self._pending_remap is not None:
            ids = torch.from_numpy(self.replica_ids.astype(np.int32)).to(self.device)
            base = self.n_local + 1
            for i in range(0, ids.numel(), chunk):
                part = ids[i:i + chunk]
                ops.gather_rows(self, part, out=self.local[base + i:base + i + part.numel(), :self.shape[1]])
            torch.cuda.synchronize()
            self.remap, self._pending_remap = self._pending_remap, None
            self._table.remap = self.remap.data_ptr()
        if self.world > 1 and dist.is_initialized():
            dist.barrier(group=self.group)

    def remote_fraction(self, ids, use_replicas=True):
        """Fraction of the given global ids whose feature row must come over NVLink (not owned; with use_replicas,
        not replicated here either)."""
        ids = ids.reshape(-1)
        own = owner_of(ids, self.n_nodes, self.world, self.row_start)
        remote = (own >= 0) & (own != self.rank)
        if use_replicas and self.remap is not None:
            safe = ids.clamp(0, self.n_nodes).long()
            remote = remote & (self.remap.to(ids.device)[safe] < 0)
        return float(remote.float().mean().item())

    def close(self):
        import torch.distributed as dist
        torch.cuda.synchronize()
        if self.world > 1 and dist.is_initialized():
            dist.barrier(group=self.group)          # nobody may still be reading our shard
        for q in self._peer_ptrs:
            check(lib().gs_ipc_close(ctypes.c_void_p(q)))
        self._peer_ptrs = []
        if self._own_ptr:
            self.local = None
            check(lib().gs_shard_free(ctypes.c_void_p(self._own_ptr)))
            self._own_ptr = None
