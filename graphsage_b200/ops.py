"""Functional wrappers: torch CUDA tensors in, torch CUDA tensors out, all work done by
libgraphsage_b200.so on the current CUDA stream.  torch only owns memory and streams here."""
import collections

import torch

from . import _lib
from ._lib import (ACT_NONE, ACT_RELU, COMBINE_ADD, COMBINE_CONCAT, MATH_FP32_SIMT, MATH_TF32X3, MATH_TF32,
                   MATH_BF16, GemmPart, GemmRowIds, RowRange, Segment, check, lib, ptr, require_cuda, stream_ptr)

_U64 = 2**64 - 1

# optional per-kernel timing (bench.py): name -> list of (start_event, end_event) on the current stream
PROBE = None
LAUNCHES = 0          # kernels of ours launched through this module (bench.py reports it as gpu_launches)
STAGE_HOOK = None     # callable(name, "pre"|"post") around probe-able launches (models.GraphedForward splits graphs here)

# The host-keyed caches (PackedWeights, PackedMlpWeights, the max-pool bf16 cast) re-pack when data_ptr() / _version say a
# tensor changed.  A replay of a captured training step (graphed_training) updates the weights without the host seeing it,
# and a capture would freeze the decision, so:
CACHE_EPOCH = [0]         # part of every cache key; advanced after each training replay
REPACK_ALWAYS = [False]   # set while a training step is captured: every call packs / casts afresh, inside the graph


def _probe(name):
    if STAGE_HOOK is not None:
        STAGE_HOOK(name, "pre")
    if PROBE is None:
        return _PostHook(name) if STAGE_HOOK is not None else None
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    PROBE.setdefault(name, []).append((e0, e1))
    e0.record()
    return e1


class _PostHook(object):
    def __init__(self, name):
        self.name = name

    def record(self):
        if STAGE_HOOK is not None:
            STAGE_HOOK(self.name, "post")


def _launched(n=1, ev=None):
    global LAUNCHES
    LAUNCHES += n
    if ev is not None:
        ev.record()


def pad_cols(f):
    return (int(f) + 7) // 8 * 8


def _i32(t, name):
    if t.dtype != torch.int32:
        raise TypeError("%s must be int32 (got %s)" % (name, t.dtype))
    return t.contiguous()


def sample_padded(adj, ids, k, seed, counter, col_perm=None, counter_dev=None, out=None):
    """UniformNeighborSampler._call - reference graphsage/neigh_samplers.py:24-29."""
    require_cuda(adj, ids, col_perm, counter_dev)
    adj, ids = _i32(adj, "adj"), _i32(ids.reshape(-1), "ids")
    n = ids.numel()
    if out is None:
        out = torch.empty((n, k), dtype=torch.int32, device=adj.device)
    ev = _probe("sample_padded")
    check(lib().gs_sample_padded(ptr(adj), adj.shape[0], adj.shape[1], ptr(ids), n, k, ptr(col_perm), seed & _U64,
                                 counter & _U64, ptr(counter_dev), ptr(out), stream_ptr()))
    _launched(1 if n * k else 0, ev)
    return out


def sample_padded_khop(adj, seeds, fanouts, seed, counter, counter_dev=None):
    """SampleAndAggregate.sample's whole frontier expansion (reference models.py:254-275) in one launch.
    fanouts in HOP order ([10, 25]); returns [hop1 ids, hop2 ids, ...] (flat int32), bit-identical to successive
    sample_padded calls with counters counter, counter+1, ..."""
    require_cuda(adj, seeds, counter_dev)
    adj, seeds = _i32(adj, "adj"), _i32(seeds.reshape(-1), "seeds")
    n = seeds.numel()
    outs, cnt = [], n
    for k in fanouts:
        cnt *= int(k)
        outs.append(torch.empty((cnt,), dtype=torch.int32, device=adj.device))
    fan = (_lib.c_i32 * len(fanouts))(*[int(k) for k in fanouts])
    optr = (_lib.c_vp * len(fanouts))(*[ptr(o) for o in outs])
    ev = _probe("sample_padded_khop")
    check(lib().gs_sample_padded_khop(ptr(adj), adj.shape[0], adj.shape[1], ptr(seeds), n, fan, len(fanouts),
                                      seed & _U64, counter & _U64, ptr(counter_dev), optr, stream_ptr()))
    _launched(1 if n else 0, ev)
    return outs


def build_padded_adj(indptr, indices, max_degree, seed=123, counter=0, skip=None):
    """Padded adjacency [N+1, max_degree] (+ degree vector) from CSR on the device - the sampler's input contract,
    reference graphsage/minibatch.py:227-259.  skip: optional bool/uint8 [N] (val/test nodes keep all-N rows)."""
    require_cuda(indptr, indices, skip)
    if indptr.dtype != torch.int64:
        raise TypeError("indptr must be int64")
    indices = _i32(indices, "indices")
    n = indptr.numel() - 1
    adj = torch.empty((n + 1, max_degree), dtype=torch.int32, device=indptr.device)
    deg = torch.empty((n,), dtype=torch.float32, device=indptr.device)
    sk = None if skip is None else skip.to(torch.uint8).contiguous()
    check(lib().gs_build_padded_adj(ptr(indptr), ptr(indices), n, max_degree, ptr(sk), seed & _U64, counter & _U64,
                                    ptr(adj), ptr(deg), stream_ptr()))
    _launched(1)
    return adj, deg


def sample_unigram(cdf, num_sampled, seed, counter, counter_dev=None):
    """tf.nn.fixed_unigram_candidate_sampler(unique=False) - reference graphsage/models.py:336-343.
    cdf: float64 CUDA tensor, inclusive prefix sum of the (distorted) unigram weights."""
    require_cuda(cdf, counter_dev)
    if cdf.dtype != torch.float64:
        raise TypeError("cdf must be float64")
    out = torch.empty((num_sampled,), dtype=torch.int32, device=cdf.device)
    check(lib().gs_sample_unigram(ptr(cdf), cdf.numel(), num_sampled, seed & _U64, counter & _U64, ptr(counter_dev),
                                  ptr(out), stream_ptr()))
    _launched(1 if num_sampled else 0)
    return out


def sample_unigram_unique(cdf, num_sampled, seed, counter, counter_dev=None, status=None):
    """tf.nn.fixed_unigram_candidate_sampler(unique=True) - reference graphsage/models.py:450-457 (Node2VecModel): the first
    num_sampled DISTINCT ids of the unigram draw sequence, in draw order (contract: oracle/node2vec.py).  cdf: float64 CUDA
    tensor, inclusive prefix sum of the weights.  The caller checks that at least num_sampled ids have positive weight
    (UniqueUnigramSampler does); if the draw budget runs out anyway the missing ids are -1 and status (an int32 CUDA
    tensor [1], optional) is set to 1."""
    require_cuda(cdf, counter_dev, status)
    if cdf.dtype != torch.float64:
        raise TypeError("cdf must be float64")
    if status is not None and (status.dtype != torch.int32 or status.numel() < 1):
        raise TypeError("status must be an int32 tensor with >= 1 element")
    if not 0 <= int(num_sampled) <= min(_lib.MAX_UNIQUE_SAMPLED, cdf.numel()):
        raise ValueError("num_sampled must be in [0, min(%d, %d)] (got %d)" % (_lib.MAX_UNIQUE_SAMPLED, cdf.numel(), num_sampled))
    out = torch.empty((num_sampled,), dtype=torch.int32, device=cdf.device)
    ev = _probe("sample_unigram_unique")
    check(lib().gs_sample_unigram_unique(ptr(cdf), cdf.numel(), int(num_sampled), seed & _U64, counter & _U64, ptr(counter_dev),
                                         ptr(out), ptr(status), stream_ptr()))
    _launched(1 if num_sampled else 0, ev)
    return out


def sample_csr(indptr, indices, ids, k, seed, counter, replace_if_short=True, pad_id=-1, counter_dev=None):
    require_cuda(indptr, indices, ids)
    if indptr.dtype != torch.int64:
        raise TypeError("indptr must be int64")
    indices, ids = _i32(indices, "indices"), _i32(ids.reshape(-1), "ids")
    n = ids.numel()
    out = torch.empty((n, k), dtype=torch.int32, device=ids.device)
    check(lib().gs_sample_csr(ptr(indptr), ptr(indices), indptr.numel() - 1, ptr(ids), n, k, int(bool(replace_if_short)),
                              seed & _U64, counter & _U64, ptr(counter_dev), pad_id, ptr(out), stream_ptr()))
    _launched(1 if n * k else 0)
    return out


def random_walks(indptr, indices, starts, num_walks, walk_len, seed, counter=0, start_offset=0):
    """Co-occurrence pairs of uniform random walks (gs_random_walks; reference graphsage/utils.py:77-92): num_walks walks
    of walk_len - 1 steps from every start, (starts[t], visited id) for every visited id other than the start, ordered
    by start, walk and step.  Contract: oracle/walks.py (start_offset is the global position of starts[0], so chunks
    with the right offsets give the pairs of one call).  Returns an int32 CUDA tensor [P, 2].
    P is read back to size the output: one device-to-host copy (and so a synchronisation) per call - start-up work,
    not meant for capture."""
    require_cuda(indptr, indices, starts)
    if indptr.dtype != torch.int64:
        raise TypeError("indptr must be int64")
    indptr, indices, starts = indptr.contiguous(), _i32(indices, "indices"), _i32(starts.reshape(-1), "starts")
    num_walks, walk_len, start_offset = int(num_walks), int(walk_len), int(start_offset)
    if not 1 <= num_walks <= _lib.WALK_MAX_WALKS:
        raise ValueError("num_walks must be in [1, %d] (got %d)" % (_lib.WALK_MAX_WALKS, num_walks))
    if not 2 <= walk_len <= _lib.WALK_MAX_LEN:
        raise ValueError("walk_len must be in [2, %d] (got %d)" % (_lib.WALK_MAX_LEN, walk_len))
    n = starts.numel()
    if not (start_offset >= 0 and start_offset + n <= 2**32):
        raise ValueError("start_offset + len(starts) must be in [0, 2^32] (got %d + %d)" % (start_offset, n))
    nbytes = lib().gs_random_walks_workspace_bytes(n, num_walks, walk_len)
    if nbytes < 0:
        check(-1)
    dev = starts.device
    ws = torch.empty((max(nbytes, 1),), dtype=torch.uint8, device=dev)
    n_pairs = torch.empty((1,), dtype=torch.int64, device=dev)
    ev = _probe("random_walks/%d" % (n * num_walks))
    check(lib().gs_random_walks(ptr(indptr), ptr(indices), indptr.numel() - 1, ptr(starts), n, num_walks, walk_len,
                                seed & _U64, counter & _U64, start_offset, ptr(ws), nbytes, ptr(n_pairs), stream_ptr()))
    out = torch.empty((int(n_pairs.item()), 2), dtype=torch.int32, device=dev)
    check(lib().gs_random_walks_emit(ptr(starts), n, num_walks, walk_len, ptr(ws), nbytes, ptr(out), stream_ptr()))
    _launched(3 if n else 0, ev)                  # walk, emit (+ CUB's scan passes)
    return out


def i8row_pitch(f):
    """Bytes per row of a GS_I8ROW table of f features (gs_i8row_pitch): round_up(round_up(f, 4) + 4, 16)."""
    return ((int(f) + 3) // 4 * 4 + 4 + 15) // 16 * 16


class I8Rows(object):
    """A GS_I8ROW table as the kernels read it (row format: include/graphsage_b200.h): `rows`, a uint8 tensor [n, pitch]
    of int8 values with each row's fp32 scale inside the row, and F features.  It stands where an fp32 [n, F] table
    would: shape (n, F), dtype torch.int8.  gather_mean, gather_rows_f32 and sage_layer_small read it as the dequantised
    fp32 table and give that table's bits."""
    dtype = torch.int8

    def __init__(self, rows, F):
        if rows.dtype != torch.uint8 or rows.dim() != 2 or rows.stride(1) != 1 or rows.stride(0) % 16 \
                or rows.shape[1] < i8row_pitch(F):
            raise ValueError("int8 rows must be a row-major uint8 [n, >= %d] tensor with a pitch of 16-byte multiples"
                             % i8row_pitch(F))
        self.rows, self.shape = rows, torch.Size((rows.shape[0], int(F)))

    @property
    def device(self):
        return self.rows.device


def _table(src):
    """(pointer, dtype code, rows, pitch) of a row-major source table: pitch in elements, or in bytes for I8Rows."""
    if isinstance(src, I8Rows):
        require_cuda(src.rows)
        return ptr(src.rows), _lib.GS_I8ROW, src.rows.shape[0], src.rows.stride(0)
    return ptr(src), _dtype_code(src), src.shape[0], src.stride(0)


def quantize_rows_i8(x, out=None):
    """fp32 [n, F] CUDA rows -> GS_I8ROW rows, uint8 [n, i8row_pitch(F)] (gs_quantize_rows_i8; contract
    oracle/int8_rows.py).  The caller refuses non-finite values."""
    require_cuda(x, out)
    if x.dtype != torch.float32 or x.dim() != 2 or x.stride(1) != 1 or x.shape[1] < 1:
        raise ValueError("x must be a row-major float32 [n, F >= 1] matrix")
    n, F = x.shape
    if out is None:
        out = torch.empty((n, i8row_pitch(F)), dtype=torch.uint8, device=x.device)
    if out.dtype != torch.uint8 or out.dim() != 2 or out.stride(1) != 1 or out.shape[0] < n or out.shape[1] != out.stride(0):
        raise ValueError("out must be a contiguous uint8 [>= n, pitch] matrix")
    check(lib().gs_quantize_rows_i8(ptr(x), n, F, x.stride(0), ptr(out), out.stride(0), stream_ptr()))
    _launched(1 if n else 0)
    return out


def _dtype_code(t):
    if t.dtype == torch.float32:
        return _lib.GS_F32
    if t.dtype == torch.bfloat16:
        return _lib.GS_BF16
    raise TypeError("features must be float32 or bfloat16 (got %s)" % t.dtype)


def gather_rows(feats, ids, out=None):
    """tf.nn.embedding_lookup(features, ids) - reference graphsage/models.py:299."""
    if hasattr(feats, "c_table"):
        ids = _i32(ids.reshape(-1), "ids")
        n, F = ids.numel(), feats.shape[1]
        if out is None:
            out = torch.empty((n, pad_cols(F)), dtype=torch.float32, device=feats.device)[:, :F]
        check(lib().gs_gather_rows_sharded(feats.c_table(), _lib.GS_F32, F, feats.pitch, ptr(ids), n, ptr(out),
                                           out.stride(0), stream_ptr()))
        _launched(1 if n else 0)
        return out
    require_cuda(feats, ids)
    if feats.dim() != 2 or feats.stride(1) != 1:
        raise ValueError("features must be a row-major 2-D tensor")
    ids = _i32(ids.reshape(-1), "ids")
    n, F = ids.numel(), feats.shape[1]
    if out is None:
        out = torch.empty((n, F), dtype=feats.dtype, device=feats.device)
    check(lib().gs_gather_rows(ptr(feats), _dtype_code(feats), feats.shape[0], F, feats.stride(0), ptr(ids), n,
                               ptr(out), out.stride(0), stream_ptr()))
    _launched(1 if n * F else 0)
    return out


def gather_rows_f32(feats, ids=None, row0=0, n=None, out=None):
    """embedding_lookup widened to fp32 (reference graphsage/models.py:299): rows ids[i] (or row0 + i) of a bf16 / fp32
    table, or of an I8Rows table (dequantised), into an fp32 [n, pad_cols(F)] buffer (returned as its [:, :F] view); pad
    columns are zeroed."""
    require_cuda(ids, out)
    if not isinstance(feats, I8Rows):
        require_cuda(feats)
        if feats.dim() != 2 or feats.stride(1) != 1:
            raise ValueError("features must be a row-major 2-D tensor")
    F = feats.shape[1]
    if ids is not None:
        ids = _i32(ids.reshape(-1), "ids")
        n = ids.numel() if n is None else int(n)
    if n is None:
        raise ValueError("n is required without ids")
    if out is None:
        out = torch.empty((n, pad_cols(F)), dtype=torch.float32, device=feats.device)[:, :F]
    if out.dtype != torch.float32 or out.stride(1) != 1 or out.shape[0] < n:
        raise ValueError("out must be a row-major float32 matrix with >= n rows")
    src, code, n_rows, pitch = _table(feats)
    check(lib().gs_gather_rows_f32(src, code, n_rows, F, pitch, ptr(ids), int(row0), n, ptr(out), out.stride(0), stream_ptr()))
    _launched(1 if n else 0)
    return out


def cast_rows_bf16(x, out=None):
    """fp32 [n, F] -> bf16 [n, pad_cols(F)] (round to nearest even, pad columns zeroed); returns the [:, :F] view."""
    require_cuda(x, out)
    if x.dtype != torch.float32 or x.dim() != 2 or x.stride(1) != 1:
        raise ValueError("x must be a row-major float32 matrix")
    n, F = x.shape
    if out is None:
        out = torch.empty((n, pad_cols(F)), dtype=torch.bfloat16, device=x.device)[:, :F]
    if out.dtype != torch.bfloat16 or out.stride(1) != 1 or out.shape[0] < n or out.stride(0) < F:
        raise ValueError("out must be a row-major bfloat16 matrix with >= n rows")
    check(lib().gs_cast_rows_bf16(ptr(x), n, F, x.stride(0), ptr(out), out.stride(0), stream_ptr()))
    _launched(1 if n else 0)
    return out


class Seg(object):
    """One hop's rows for gather_mean: n output rows with fanout k.  Neighbour j of row i is
    src[neigh_ids[i*k + j]] (or src[neigh_row0 + i*k + j] when neigh_ids is None); the self row is
    src[self_ids[i]] (or src[self_row0 + i]).  Output row = out_row0 + i."""
    __slots__ = ("n", "k", "self_ids", "neigh_ids", "self_row0", "neigh_row0", "out_row0")

    def __init__(self, n, k, self_ids=None, neigh_ids=None, self_row0=0, neigh_row0=0, out_row0=0):
        self.n, self.k = int(n), int(k)
        self.self_ids = None if self_ids is None else _i32(self_ids.reshape(-1), "self_ids")
        self.neigh_ids = None if neigh_ids is None else _i32(neigh_ids.reshape(-1), "neigh_ids")
        self.self_row0, self.neigh_row0, self.out_row0 = int(self_row0), int(neigh_row0), int(out_row0)
        if self.self_ids is not None and self.self_ids.numel() < self.n:
            raise ValueError("self_ids shorter than n")
        if self.neigh_ids is not None and self.neigh_ids.numel() < self.n * self.k:
            raise ValueError("neigh_ids shorter than n*k")

    def c_struct(self):
        require_cuda(self.self_ids, self.neigh_ids)
        return Segment(ptr(self.self_ids), ptr(self.neigh_ids), self.self_row0, self.neigh_row0, self.n, self.k, 0,
                       self.out_row0)


def make_segment(n, k, self_ids=None, neigh_ids=None, self_row0=0, neigh_row0=0, out_row0=0):
    return Seg(n, k, self_ids, neigh_ids, self_row0, neigh_row0, out_row0)



def _check_out(t, rows, out_pitch, name):
    """A caller-provided output of gather_mean: the library writes rows x out_pitch floats at row stride out_pitch."""
    if t is None:
        return
    require_cuda(t)
    if t.dtype != torch.float32 or t.dim() != 2 or t.stride(1) != 1 or t.stride(0) != out_pitch or t.shape[0] < rows:
        raise ValueError("%s must be a float32 [>= %d, .] CUDA matrix with row stride out_pitch = %d" % (name, rows, out_pitch))


def gather_mean(src, segments, include_self=False, want_self=True, out_pitch=None, out_mean=None, out_self=None):
    """Fused embedding_lookup + reduce_mean over the fanout (models.py:299 + aggregators.py:48 / :106-107).
    segments: list of Seg; returns (out_self or None, out_mean), each [rows, out_pitch].
    `src` is a float32 (or bfloat16) [rows, F] CUDA tensor, an I8Rows table (the means of its dequantised rows), or a
    parallel.ShardedFeatures (node-partitioned table)."""
    if hasattr(src, "c_table"):
        return _gather_mean_sharded(src, segments, include_self, want_self, out_pitch, out_mean, out_self)
    if not isinstance(src, I8Rows):
        require_cuda(src)
        if src.dtype not in (torch.float32, torch.bfloat16) or src.dim() != 2 or src.stride(1) != 1:
            raise ValueError("src must be a row-major float32 (or bfloat16) 2-D tensor")
    F = src.shape[1]
    if out_pitch is None:
        out_pitch = pad_cols(F)
    rows = max([s.out_row0 + s.n for s in segments] + [0])
    _check_out(out_mean, rows, out_pitch, "out_mean")
    _check_out(out_self if want_self else None, rows, out_pitch, "out_self")
    if out_mean is None:
        out_mean = torch.empty((rows, out_pitch), dtype=torch.float32, device=src.device)
    if want_self and out_self is None:
        out_self = torch.empty((rows, out_pitch), dtype=torch.float32, device=src.device)
    arr = (Segment * max(len(segments), 1))(*[s.c_struct() for s in segments])
    ev = _probe("gather_mean/%d" % rows)
    table, code, n_rows, pitch = _table(src)
    check(lib().gs_gather_mean(table, code, n_rows, F, pitch, arr, len(segments),
                               int(bool(include_self)), ptr(out_self) if want_self else 0, ptr(out_mean), out_pitch,
                               stream_ptr()))
    _launched(1 if rows else 0, ev)
    return (out_self if want_self else None), out_mean


def translate_ids(table, ids):
    """ids -> locators of a parallel.ShardedFeatures with replicas (gs_translate_ids): >= 0 a row of this GPU's own buffer,
    < 0 -> -(global id) - 1 (the row has to come from its owner)."""
    ids = _i32(ids.reshape(-1), "ids")
    out = torch.empty_like(ids)
    check(lib().gs_translate_ids(table.c_table(), ptr(ids), ids.numel(), ptr(out), stream_ptr()))
    _launched(1 if ids.numel() else 0)
    return out


def host_register(t):
    """Page-lock a contiguous CPU tensor once and map it for the device (gs_host_register); returns its device alias."""
    import ctypes
    if t.is_cuda or not t.is_contiguous():
        raise ValueError("host_register needs a contiguous CPU tensor")
    alias = ctypes.c_void_p()
    check(lib().gs_host_register(t.data_ptr(), t.numel() * t.element_size(), ctypes.byref(alias)))
    return alias.value


def host_unregister(t):
    check(lib().gs_host_unregister(t.data_ptr()))


def host_fetch(host_alias, row_bytes, stage_ids, count, staging):
    """staging[i] = row stage_ids[i] of the mapped host table, i < *count (gs_host_fetch); staging rows are row_bytes
    apart, the table's pitch.  capacity = stage_ids.numel(); the launch does not read *count on the host."""
    capacity = stage_ids.numel()
    ev = _probe("host_fetch")
    check(lib().gs_host_fetch(host_alias, int(row_bytes), ptr(stage_ids), ptr(count), capacity, ptr(staging),
                              stream_ptr()))
    _launched(1 if capacity else 0, ev)


def host_translate(table, ids, claim, stage_row0, out=None):
    """ids -> working-set rows of a host table (gs_host_translate): the cache slot, the zero row, or stage_row0 + slot."""
    ids = _i32(ids.reshape(-1), "ids")
    if out is None:
        out = torch.empty_like(ids)
    check(lib().gs_host_translate(table, ptr(ids), ids.numel(), ptr(claim), int(stage_row0), ptr(out), stream_ptr()))
    _launched(1 if ids.numel() else 0)
    return out


def _shard_prepare(src, segments):
    """Row addressing for a gather over a parallel.ShardedFeatures: returns (segments, ids_are_locators, staging)."""
    F = src.shape[1]
    locators, staging = 0, None
    by_ids = any(s.self_ids is not None or s.neigh_ids is not None for s in segments)
    if by_ids and src.world > 1 and getattr(src, "stage_halo", True):
        # halo staging: every remote row of the step crosses NVLink once (claim -> fetch -> translate), then the gather
        # reads local memory only.  All buffers are per call: under CUDA-graph capture they live in the graph's pool.
        lists, order = {}, []
        for s in segments:
            if s.self_ids is None or s.neigh_ids is None:
                raise ValueError("with halo staging every segment of a sharded gather must address its rows by ids")
            for t in (s.self_ids, s.neigh_ids):
                key = (t.data_ptr(), t.numel())
                if key not in lists:
                    lists[key] = t
                    order.append(key)
        capacity = sum(lists[k].numel() for k in order)
        dev = src.device
        claim = torch.empty((src.shape[0],), dtype=torch.int32, device=dev)
        count = torch.empty((1,), dtype=torch.int32, device=dev)
        stage_ids = torch.empty((capacity,), dtype=torch.int32, device=dev)
        staging = torch.empty((capacity, src.pitch), dtype=torch.float32, device=dev)
        check(lib().gs_halo_begin(ptr(claim), src.shape[0], ptr(count), stream_ptr()))
        for k in order:
            check(lib().gs_halo_claim(src.c_table(), ptr(lists[k]), lists[k].numel(), ptr(claim), ptr(count), ptr(stage_ids),
                                      capacity, stream_ptr()))
        check(lib().gs_halo_fetch(src.c_table(), F, src.pitch, ptr(stage_ids), ptr(count), capacity, ptr(staging), src.pitch,
                                  stream_ptr()))
        locs = {}
        for k in order:
            locs[k] = torch.empty_like(lists[k])
            check(lib().gs_halo_translate(src.c_table(), ptr(lists[k]), lists[k].numel(), ptr(claim), ptr(locs[k]), stream_ptr()))
        _launched(2 * len(order) + 1)
        segments = [Seg(s.n, s.k, locs[(s.self_ids.data_ptr(), s.self_ids.numel())],
                        locs[(s.neigh_ids.data_ptr(), s.neigh_ids.numel())], s.self_row0, s.neigh_row0, s.out_row0)
                    for s in segments]
        locators = 2
    elif by_ids and getattr(src, "remap", None) is not None:
        # replicas, no staging: resolve every id list once (one pass per distinct tensor; hop-1 ids are self ids of one
        # segment and neighbour ids of another) so the gather kernel's issue path has no table lookup
        done, segs = {}, []

        def tr(t):
            key = (t.data_ptr(), t.numel())
            if key not in done:
                done[key] = translate_ids(src, t)
            return done[key]

        for s in segments:
            # locators are row indices of this GPU's buffer: a row-range segment in the same call would be read as such
            if s.self_ids is None or s.neigh_ids is None:
                raise ValueError("with replicas every segment of a sharded gather must address its rows by ids")
            segs.append(Seg(s.n, s.k, tr(s.self_ids), tr(s.neigh_ids), s.self_row0, s.neigh_row0, s.out_row0))
        segments, locators = segs, 1
    return segments, locators, staging


def _gather_mean_sharded(src, segments, include_self, want_self, out_pitch, out_mean, out_self):
    F = src.shape[1]
    if out_pitch is None:
        out_pitch = pad_cols(F)
    rows = max([s.out_row0 + s.n for s in segments] + [0])
    _check_out(out_mean, rows, out_pitch, "out_mean")
    _check_out(out_self if want_self else None, rows, out_pitch, "out_self")
    if out_mean is None:
        out_mean = torch.empty((rows, out_pitch), dtype=torch.float32, device=src.device)
    if want_self and out_self is None:
        out_self = torch.empty((rows, out_pitch), dtype=torch.float32, device=src.device)
    segments, locators, staging = _shard_prepare(src, segments)
    arr = (Segment * max(len(segments), 1))(*[s.c_struct() for s in segments])
    ev = _probe("gather_mean/%d" % rows)
    check(lib().gs_gather_mean_sharded(src.c_table(), _lib.GS_F32, F, src.pitch, arr, len(segments),
                                       int(bool(include_self)), locators, ptr(staging), ptr(out_self) if want_self else 0,
                                       ptr(out_mean), out_pitch, stream_ptr()))
    _launched(1 if rows else 0, ev)
    return (out_self if want_self else None), out_mean


def segment_max(x, n, k):
    require_cuda(x)
    C = x.shape[1]
    out = torch.empty((n, C), dtype=torch.float32, device=x.device)
    check(lib().gs_segment_max(ptr(x), n, k, C, x.stride(0), ptr(out), out.stride(0), stream_ptr()))
    _launched(1 if n * C else 0)
    return out


CSR_OPS = {"mean": _lib.CSR_MEAN, "mean_self": _lib.CSR_MEAN_SELF, "max": _lib.CSR_MAX, "sum": _lib.CSR_SUM}


def csr_aggregate(src, indptr, indices, op, rows=None, out=None, dropout=None, t_slot=None):
    """The reduction of each node's whole CSR row (gs_csr_aggregate; contract in oracle/full_neighbor.py): output row i is
    for node v = rows[i] - or, without rows, for every node 0 .. N-1 and then the dummy node N (N = len(indptr) - 1: the
    [N+1, .] layout of the tables it reads) - over the source rows indices[indptr[v] .. indptr[v+1]) in CSR order - op "mean", "mean_self"
    (GCN: v's own row joins the sum, divisor count + 1) or "max".  An empty row, or v outside [0, len(indptr) - 1), reduces
    over the last source row (the dummy) alone; entries outside the table read it too.  op "sum" (fp32 src only): the plain
    sum in CSR order, +0 for an empty row - the backward of the means over csr_transpose's graph
    (oracle/full_neighbor_grad.py); its CSR has one row per source row (len(indptr) = R + 1), and without rows the output
    is those R rows, with no extra dummy row.  src: fp32 or bf16 [R, F] CUDA table.  Returns fp32 [n, F], a view of an
    [n, pad_cols(F)] buffer (or of `out`, whose extra columns are zeroed).
    dropout: None, or (neighbour site, self site, (pos_indptr, pos_ids or None, pos_nnz)) - full-neighbourhood training
    dropout (gs_csr_aggregate_dropout; contract in oracle/full_neighbor_dropout.py) for ops "mean", "mean_self" and "sum";
    "sum" then also takes t_slot, the slots of csr_transpose(..., slots=True)."""
    require_cuda(src, indptr, indices, rows, out)
    if src.dtype not in (torch.float32, torch.bfloat16) or src.dim() != 2 or src.stride(1) != 1:
        raise ValueError("src must be a row-major float32 (or bfloat16) 2-D tensor")
    if indptr.dtype != torch.int64 or indptr.dim() != 1 or indptr.numel() < 1:
        raise TypeError("indptr must be a 1-D int64 tensor with >= 1 element")
    if op not in CSR_OPS:
        raise ValueError("op must be one of %s (got %r)" % (sorted(CSR_OPS), op))
    if op == "sum" and src.dtype != torch.float32:
        raise ValueError("op 'sum' reads float32 sources only")
    if op == "sum" and indptr.numel() != src.shape[0] + 1:
        # the sum runs over a square graph such as csr_transpose's: one CSR row per source row (the forward CSR of an
        # [N+1, .] table has only N)
        raise ValueError("op 'sum' needs one CSR row per source row: indptr of %d entries for %d source rows (got %d) - "
                         "the layout of csr_transpose" % (src.shape[0] + 1, src.shape[0], indptr.numel()))
    indptr, indices = indptr.contiguous(), _i32(indices.reshape(-1), "indices")
    if indices.numel() == 0:
        indices = torch.zeros((1,), dtype=torch.int32, device=indptr.device)
    n_nodes = indptr.numel() - 1
    if rows is not None:
        rows = _i32(rows.reshape(-1), "rows")
    n, F = (n_nodes + (op != "sum") if rows is None else rows.numel()), src.shape[1]
    if out is None:
        out = torch.empty((n, pad_cols(F)), dtype=torch.float32, device=src.device)
    if out.dtype != torch.float32 or out.dim() != 2 or out.stride(1) != 1 or out.shape[0] < n:
        raise ValueError("out must be a row-major float32 [>= %d, .] CUDA matrix" % n)
    if dropout is not None:
        neigh, self_site, (pos_indptr, pos_ids, pos_nnz) = dropout
        if op == "max":
            raise ValueError("dropout applies to the ops 'mean', 'mean_self' and 'sum'")
        if op == "sum" and (t_slot is None or t_slot.dtype != torch.int32 or t_slot.numel() < indices.numel()):
            raise ValueError("op 'sum' with dropout needs t_slot, int32 with one slot per transposed entry")
        require_cuda(pos_indptr, pos_ids, t_slot)
        if pos_indptr.dtype != torch.int64 or pos_indptr.dim() != 1:
            raise TypeError("pos_indptr must be a 1-D int64 tensor")
        if pos_ids is not None:
            pos_ids = _i32(pos_ids.reshape(-1), "pos_ids")
            need = n_nodes if op == "sum" else n_nodes + 1         # the sum's CSR has a row per source row already
            if pos_ids.numel() < need:
                raise ValueError("pos_ids needs one id per local row: %d, got %d" % (need, pos_ids.numel()))
        ev = _probe("csr_aggregate_dropout/%d" % n)
        check(lib().gs_csr_aggregate_dropout(ptr(src), _dtype_code(src), src.shape[0], F, src.stride(0), ptr(indptr),
                                             ptr(indices), ptr(t_slot) if op == "sum" else 0, n_nodes, ptr(rows), n,
                                             CSR_OPS[op], dropout_site(neigh), dropout_site(self_site),
                                             ptr(pos_indptr.contiguous()), ptr(pos_ids), int(pos_nnz), ptr(out),
                                             out.stride(0), stream_ptr()))
        _launched(1 if n else 0, ev)
        return out[:n, :F]
    ev = _probe("csr_aggregate/%d" % n)
    check(lib().gs_csr_aggregate(ptr(src), _dtype_code(src), src.shape[0], F, src.stride(0), ptr(indptr), ptr(indices),
                                 n_nodes, ptr(rows), n, CSR_OPS[op], ptr(out), out.stride(0), stream_ptr()))
    _launched(1 if n else 0, ev)
    return out[:n, :F]


def _csr_args(indptr, indices):
    require_cuda(indptr, indices)
    if indptr.dtype != torch.int64 or indptr.dim() != 1 or indptr.numel() < 1:
        raise TypeError("indptr must be a 1-D int64 tensor with >= 1 element")
    return indptr.contiguous(), _i32(indices.reshape(-1), "indices")


def csr_transpose(indptr, indices, with_self=False, slots=False):
    """The transpose of the effective CSR of the full-neighbourhood forward (gs_csr_transpose; contract in
    oracle/full_neighbor_grad.py): over N + 1 rows (N = len(indptr) - 1), entries outside [0, N] read as N, an empty row and
    the dummy row N as {N}, with_self (GCN) appending each row's own id.  Row j of the result lists, in ascending order,
    the rows i with an entry j (once per entry).  Returns (t_indptr int64 [N + 2], t_indices int32 [capacity]): entries
    past t_indptr[-1] are unspecified.  Built on the device - the entry count is not read back.  slots: also return
    t_slot int32 [capacity], where each transposed entry sits in its forward row (j, -1 for the implicit {N} entry, -2 for
    the with_self entry) - what the masked backward sum reads; t_indptr and t_indices are the same bytes."""
    indptr, indices = _csr_args(indptr, indices)
    n_nodes, nnz, ws_self = indptr.numel() - 1, indices.numel(), int(bool(with_self))
    nbytes = lib().gs_csr_transpose_workspace_bytes(n_nodes, nnz, ws_self)
    if nbytes < 0:
        check(-1)
    cap = nnz + (n_nodes + 1) * (1 + ws_self)
    t_indptr = torch.empty((n_nodes + 2,), dtype=torch.int64, device=indptr.device)
    t_indices = torch.empty((cap,), dtype=torch.int32, device=indptr.device)
    t_slot = torch.empty((cap,), dtype=torch.int32, device=indptr.device) if slots else None
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=indptr.device)
    ev = _probe("csr_transpose/%d" % cap)
    check(lib().gs_csr_transpose(ptr(indptr), ptr(indices) if nnz else 0, n_nodes, nnz, ws_self, ptr(t_indptr),
                                 ptr(t_indices), ptr(t_slot), ptr(ws), nbytes, stream_ptr()))
    _launched(5 if slots else 4, ev)     # counts, fill, indptr (+ CUB's scan and sort passes), slots
    return (t_indptr, t_indices, t_slot) if slots else (t_indptr, t_indices)


def csr_max_backward(z, m, dm, indptr, indices, t_indptr, t_indices, s=None, out=None):
    """The gradient of m = csr_aggregate(z, indptr, indices, "max") over all N + 1 rows, through the ReLU that made z
    (gs_csr_max_backward; oracle/full_neighbor_grad.py): s = dm / tie count per (row, column), then per node j the sum, in
    transposed order, of s[i] over the rows i that read j where z[j] attains m[i]; +0 where z[j] <= 0.  z, m, dm: fp32
    [N + 1, F] CUDA matrices with unit column stride; (t_indptr, t_indices) = csr_transpose(indptr, indices).  s: optional
    [N + 1, >= F] scratch (the scale of phase (a), kept for inspection).  Returns fp32 [N + 1, F]."""
    indptr, indices = _csr_args(indptr, indices)
    t_indptr, t_indices = _csr_args(t_indptr, t_indices)
    rows = indptr.numel()
    if t_indptr.numel() != rows + 1:
        raise ValueError("t_indptr must have N + 2 = %d entries" % (rows + 1))
    for name, t in (("z", z), ("m", m), ("dm", dm)):
        _fp32_table(t, name, 1)
        if t.shape[0] != rows:
            raise ValueError("%s must have N + 1 = %d rows" % (name, rows))
    F = z.shape[1]
    if m.shape[1] != F or dm.shape[1] != F:
        raise ValueError("z, m and dm must have the same width")
    if s is None:
        s = torch.empty((rows, pad_cols(F)), dtype=torch.float32, device=z.device)
    if out is None:
        out = torch.empty((rows, pad_cols(F)), dtype=torch.float32, device=z.device)
    for name, t in (("s", s), ("out", out)):
        _fp32_table(t, name, F)
        if t.shape[0] != rows:
            raise ValueError("%s must have N + 1 = %d rows" % (name, rows))
    if indices.numel() == 0:
        indices = torch.zeros((1,), dtype=torch.int32, device=indptr.device)
    ev = _probe("csr_max_backward/%d" % rows)
    check(lib().gs_csr_max_backward(ptr(z), z.stride(0), ptr(m), m.stride(0), ptr(dm), dm.stride(0), F, ptr(indptr),
                                    ptr(indices), ptr(t_indptr), ptr(t_indices), rows - 1, ptr(s), s.stride(0), ptr(out),
                                    out.stride(0), stream_ptr()))
    _launched(2, ev)
    return out[:, :F]


CsrBlock = collections.namedtuple("CsrBlock", ["src_ids", "indptr", "indices", "rows"])   # one layer of csr_blocks


def csr_blocks(indptr, indices, seeds, n_layers):
    """The receptive field of `seeds` over n_layers layers of whole neighbourhoods (gs_csr_blocks_plan / _fill; contract
    in oracle/full_neighbor_blocks.py): a list, index l = layer l, of CsrBlock(src_ids int32 V_l, indptr int64 [|V_l|],
    indices int32, rows int32).  A block is a CSR over |V_l| - 1 local nodes whose last local row is the dummy, so
    csr_aggregate(table of V_l's rows, indptr, indices, rows=rows) gives the whole-graph layer's rows of the next level.
    Built on the device; the 2L sizes are read back once to allocate the outputs - one device-to-host copy (and so a
    synchronisation) per call, not meant for capture."""
    require_cuda(indptr, indices, seeds)
    if indptr.dtype != torch.int64 or indptr.dim() != 1 or indptr.numel() < 1:
        raise TypeError("indptr must be a 1-D int64 tensor with >= 1 element")
    indptr, indices, seeds = indptr.contiguous(), _i32(indices.reshape(-1), "indices"), _i32(seeds.reshape(-1), "seeds")
    L = int(n_layers)
    if not 1 <= L <= _lib.MAX_BLOCK_LAYERS:
        raise ValueError("n_layers must be in [1, %d] (got %d)" % (_lib.MAX_BLOCK_LAYERS, L))
    n_nodes, nnz, n = indptr.numel() - 1, indices.numel(), seeds.numel()
    nbytes = lib().gs_csr_blocks_workspace_bytes(n_nodes, nnz, n, L)
    if nbytes < 0:
        check(-1)
    dev = indptr.device
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
    counts = torch.empty((2 * L,), dtype=torch.int64, device=dev)
    ev = _probe("csr_blocks/%d" % n)
    check(lib().gs_csr_blocks_plan(ptr(indptr), ptr(indices) if nnz else 0, n_nodes, nnz, ptr(seeds) if n else 0, n, L,
                                   ptr(ws), nbytes, ptr(counts), stream_ptr()))
    sizes = [int(x) for x in counts.tolist()]                # the one device-to-host read
    out_rows = [sizes[2 * l + 2] for l in range(L - 1)] + [n]
    blocks = [CsrBlock(torch.empty((sizes[2 * l],), dtype=torch.int32, device=dev),
                       torch.empty((sizes[2 * l],), dtype=torch.int64, device=dev),
                       torch.empty((sizes[2 * l + 1],), dtype=torch.int32, device=dev),
                       torch.empty((out_rows[l],), dtype=torch.int32, device=dev)) for l in range(L)]
    arrs = [(_lib.c_vp * L)(*[ptr(b[k]) if b[k].numel() else 0 for b in blocks]) for k in range(4)]
    check(lib().gs_csr_blocks_fill(ptr(indptr), ptr(indices) if nnz else 0, n_nodes, nnz, ptr(seeds) if n else 0, n, L,
                                   ptr(ws), nbytes, (_lib.c_i64 * (2 * L))(*sizes), *arrs, stream_ptr()))
    _launched(6 * L + 4, ev)           # plan: mark, compact, size, degrees per level; fill: degrees, fill, rows (+ CUB)
    return blocks


class TableRows(object):
    """A sage_gemm A operand of M rows read by id from a row table (gs_sage_gemm_rows), for rows that only feed the GEMM:
    for each (ids, row0) of `ranges`, operand row row0 + i is table[ids[i]].  Ids outside [0, table rows) read the table's
    last row (the zero dummy row), rows no range covers are zero.  The result equals sage_gemm on the gathered rows, bit for
    bit, in every math."""
    __slots__ = ("table", "ranges", "M")

    def __init__(self, table, ranges, M):
        require_cuda(table)
        if table.dtype != torch.float32 or table.dim() != 2 or table.stride(1) != 1:
            raise ValueError("the row table must be a row-major float32 matrix")
        if len(ranges) > _lib.MAX_SEGMENTS:
            raise ValueError("at most %d id ranges" % _lib.MAX_SEGMENTS)
        self.table, self.M = table, int(M)
        self.ranges = [(_i32(ids.reshape(-1), "ids"), int(row0)) for ids, row0 in ranges]
        require_cuda(*[ids for ids, _ in self.ranges])

    @property
    def device(self):
        return self.table.device

    def c_struct(self):
        r = GemmRowIds(self.table.shape[0], len(self.ranges), 0)
        for s, (ids, row0) in enumerate(self.ranges):
            r.ranges[s] = RowRange(ptr(ids), row0, ids.numel())
        return r


def _gemm_parts(parts):
    A0 = parts[0][0]
    M = A0.M if isinstance(A0, TableRows) else (A0.shape[0] if A0 is not None else 0)
    arr = (GemmPart * len(parts))()
    keep = []
    for i, (A, K, B) in enumerate(parts):
        by_id = isinstance(A, TableRows)
        if by_id:
            if A.M != M:
                raise ValueError("bad A operand for part %d" % i)
            A = A.table
        require_cuda(A, B)
        if (A is not None and A.dtype != torch.float32) or B.dtype != torch.float32:
            raise TypeError("sage_gemm operands must be float32")
        if A is not None and (A.stride(1) != 1 or (A.shape[0] != M and not by_id) or A.shape[1] < K):
            raise ValueError("bad A operand for part %d" % i)
        B = B.contiguous()
        if B.shape[0] != K:
            raise ValueError("part %d: B has %d rows, expected K=%d" % (i, B.shape[0], K))
        keep.append(B)
        arr[i] = GemmPart(ptr(A), A.stride(0) if A is not None else K, K, ptr(B), B.stride(0), B.shape[1])
    return M, arr, keep


class PackedWeights(object):
    """Tensor-core weight images cached across calls (inference: the weights do not change between steps).
    Re-packed automatically when a weight tensor is replaced or modified in place."""

    def __init__(self):
        self.key, self.ws = None, None

    def get(self, parts, arr, math, dev):
        if REPACK_ALWAYS[0]:                     # captured: the pack is part of the graph, into a buffer of its pool
            return self._pack(parts, arr, math, dev, None)
        key = (CACHE_EPOCH[0], math) + tuple((p[2].data_ptr(), p[2]._version, tuple(p[2].shape)) for p in parts)
        if key != self.key:
            self.ws = self._pack(parts, arr, math, dev, self.ws)
            self.key = key
        return self.ws

    @staticmethod
    def _pack(parts, arr, math, dev, ws):
        nbytes = lib().gs_sage_gemm_workspace_bytes(1, arr, len(parts), math)
        if nbytes < 0:
            check(-1)
        if ws is None or ws.numel() < nbytes:
            ws = torch.empty((max(nbytes, 1),), dtype=torch.uint8, device=dev)
        check(lib().gs_sage_gemm_pack(arr, len(parts), math, ptr(ws), stream_ptr()))
        _launched(1)
        return ws


def sage_gemm(parts, combine=COMBINE_ADD, bias=None, act=ACT_NONE, math=MATH_FP32_SIMT, out=None, packed=None):
    """parts: [(A[M, >=K] (row stride used as lda) or a TableRows, K, B[K, N])] (1 or 2).
    act(concat_or_add(A_p[:, :K] @ B_p) + bias).
    packed: optional PackedWeights cache (tensor-core modes) so the weight images are built once, not per call."""
    M, arr, keep = _gemm_parts(parts)
    rid = None
    if any(isinstance(p[0], TableRows) for p in parts):
        rid = (GemmRowIds * len(parts))()
        for i, p in enumerate(parts):
            if isinstance(p[0], TableRows):
                rid[i] = p[0].c_struct()
    ntot = sum(p[2].shape[1] for p in parts) if (combine == COMBINE_CONCAT) else parts[0][2].shape[1]
    dev = parts[0][0].device
    if out is None:
        out = torch.empty((M, ntot), dtype=torch.float32, device=dev)

    def run(ws):
        if rid is None:
            return lib().gs_sage_gemm_prepacked(M, arr, len(parts), combine, ptr(bias), act, math, ptr(out), out.stride(0),
                                                ptr(ws), stream_ptr())
        return lib().gs_sage_gemm_rows(M, arr, rid, len(parts), combine, ptr(bias), act, math, ptr(out), out.stride(0),
                                       ptr(ws), stream_ptr())

    if math == MATH_FP32_SIMT or packed is None:
        ws_bytes = lib().gs_sage_gemm_workspace_bytes(M, arr, len(parts), math)
        if ws_bytes < 0:
            check(-1)
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev) if ws_bytes > 0 else None
        ev = _probe("sage_gemm/%d" % M)
        if M and ws is not None:             # gs_sage_gemm = pack + prepacked
            check(lib().gs_sage_gemm_pack(arr, len(parts), math, ptr(ws), stream_ptr()))
        check(run(ws))
        _launched((2 if ws is not None else 1) if M else 0, ev)
        return out
    ws = packed.get(parts, arr, math, dev)
    ev = _probe("sage_gemm/%d" % M)
    check(run(ws))
    _launched(1 if M else 0, ev)
    return out


SMALL_LAYER_MAX_ROWS = 2048


def sage_layer_small(src, seg, parts, combine=COMBINE_ADD, include_self=False, bias=None, act=ACT_NONE,
                     l2_normalize=False, counter_dev=None, counter_inc=0):
    """One whole aggregator layer (fanout mean -> matmuls -> add|concat -> bias -> act -> optional row
    l2-normalise) for a small number of rows in ONE launch, exact fp32.  parts: [(None, K, B)] with K == src width.
    src: a float32 CUDA table, or an I8Rows table (gs_sage_layer_small_i8: the bits of the dequantised table)."""
    require_cuda(bias, counter_dev)
    i8 = isinstance(src, I8Rows)
    if not i8:
        require_cuda(src)
        if src.dtype != torch.float32 or src.stride(1) != 1:
            raise ValueError("src must be row-major float32")
    _, arr, keep = _gemm_parts([(None, K, B) for (_, K, B) in parts])
    ntot = sum(p[2].shape[1] for p in parts) if (combine == COMBINE_CONCAT) else parts[0][2].shape[1]
    rows = seg.out_row0 + seg.n
    out = torch.empty((rows, ntot), dtype=torch.float32, device=src.device)
    cseg = seg.c_struct()
    ev = _probe("sage_layer_small/%d" % rows)
    table, _, n_rows, pitch = _table(src)
    fn = lib().gs_sage_layer_small_i8 if i8 else lib().gs_sage_layer_small
    check(fn(table, n_rows, src.shape[1], pitch, cseg, int(bool(include_self)), arr, len(parts), combine, ptr(bias), act,
             int(bool(l2_normalize)), ptr(out), out.stride(0), ptr(counter_dev), int(counter_inc), stream_ptr()))
    _launched(1 if seg.n else 0, ev)
    return out


class PackedMlpWeights(object):
    """bf16 tile images of the max-pool MLP weight for gs_maxpool_mlp_fused, re-packed when the weight changes."""

    def __init__(self):
        self.key, self.ws = None, None

    def get(self, W):
        if REPACK_ALWAYS[0]:
            return self._pack(W)
        key = (CACHE_EPOCH[0], W.data_ptr(), W._version, tuple(W.shape))
        if key != self.key:
            self.ws = self._pack(W)
            self.key = key
        return self.ws

    @staticmethod
    def _pack(W):
        K, hidden = W.shape
        nbytes = lib().gs_maxpool_mlp_workspace_bytes(K, hidden)
        ws = torch.empty((nbytes,), dtype=torch.uint8, device=W.device)
        Wc = W.contiguous()
        check(lib().gs_maxpool_mlp_pack(ptr(Wc), Wc.stride(0), K, hidden, ptr(ws), stream_ptr()))
        _launched(1)
        return ws


def _check_mlp_K(W, K):
    """The K columns the fused pooling kernels read: the packed images hold ceil(W.shape[0] / 64) K-blocks of W and the
    kernels walk ceil(K / 64), so K must be at most W's row count and within its last K-block."""
    if K is None:
        return W.shape[0]
    if not 1 <= K <= W.shape[0] or (K + 63) // 64 != (W.shape[0] + 63) // 64:
        raise ValueError("K = %d does not match the MLP weight's %d rows (K <= rows, the same number of 64-column "
                         "blocks)" % (K, W.shape[0]))
    return K


def maxpool_mlp_fused(table, n_groups, k, W, bias, packed, row_ids=None, row0=0, K=None, out=None, pool="max"):
    """out[g, :] = max_j relu(table[row(g, j), :K] @ W + bias) in one wgmma kernel (bf16 operands, fp32 accumulate).
    table: bfloat16 [rows, >=K] row-major with pitch % 8 == 0; W: float32 [K, hidden] (hidden % 128 == 0)."""
    require_cuda(table, W, bias, row_ids)
    if table.dtype != torch.bfloat16 or table.stride(1) != 1:
        raise TypeError("table must be row-major bfloat16")
    K = _check_mlp_K(W, K)
    hidden = W.shape[1]
    if out is None:
        out = torch.empty((n_groups, hidden), dtype=torch.float32, device=table.device)
    ws = packed.get(W)
    if row_ids is not None:
        row_ids = _i32(row_ids.reshape(-1), "row_ids")
    ev = _probe("maxpool_mlp/%d" % n_groups)
    fn = lib().gs_meanpool_mlp_fused if pool == "mean" else lib().gs_maxpool_mlp_fused
    check(fn(ptr(table), table.shape[0], K, table.stride(0), ptr(row_ids), row0, n_groups, k,
             ptr(ws), ptr(bias), hidden, ptr(out), out.stride(0), stream_ptr()))
    _launched(1 if n_groups else 0, ev)
    return out


def maxpool2_mlp_fused(table, n_groups, k, W1, b1, packed1, W2, b2, packed2, row_ids=None, row0=0, K=None, out=None):
    """out[g, :] = max_j relu(bf16(relu(table[row(g, j), :K] @ W1 + b1)) @ W2 + b2) in one wgmma kernel (K5; bf16
    operands, fp32 accumulate; contract: oracle/pool2_forward.py).  table: bfloat16 [rows, >=K] row-major with
    pitch % 8 == 0; W1: float32 [K, h1] (h1 % 128 == 0); W2: float32 [h1, h2] (h2 % 256 == 0); packed1 / packed2:
    PackedMlpWeights, one per weight."""
    require_cuda(table, W1, b1, W2, b2, row_ids)
    if table.dtype != torch.bfloat16 or table.stride(1) != 1:
        raise TypeError("table must be row-major bfloat16")
    K = _check_mlp_K(W1, K)
    h1, h2 = W1.shape[1], W2.shape[1]
    if W2.shape[0] != h1:
        raise ValueError("W2 must have h1 = %d rows (got %d)" % (h1, W2.shape[0]))
    if out is None:
        out = torch.empty((n_groups, h2), dtype=torch.float32, device=table.device)
    ws1, ws2 = packed1.get(W1), packed2.get(W2)
    if row_ids is not None:
        row_ids = _i32(row_ids.reshape(-1), "row_ids")
    ev = _probe("maxpool2_mlp/%d" % n_groups)
    check(lib().gs_maxpool2_mlp_fused(ptr(table), table.shape[0], K, table.stride(0), ptr(row_ids), row0, n_groups, k,
                                      ptr(ws1), ptr(b1), h1, ptr(ws2), ptr(b2), h2, ptr(out), out.stride(0), stream_ptr()))
    _launched(1 if n_groups else 0, ev)
    return out


class PackedMlpDxWeights(PackedMlpWeights):
    """bf16 images of Wm[:cols] (K-major over hidden) for pool_mlp_backward_dx, re-packed when the weight changes."""

    def __init__(self, cols):
        PackedMlpWeights.__init__(self)
        self.cols = int(cols)

    def get(self, W):
        if REPACK_ALWAYS[0]:
            return self._pack_dx(W, self.cols)
        key = (CACHE_EPOCH[0], W.data_ptr(), W._version, tuple(W.shape), self.cols)
        if key != self.key:
            self.ws = self._pack_dx(W, self.cols)
            self.key = key
        return self.ws

    @staticmethod
    def _pack_dx(W, cols):
        if not 1 <= cols <= W.shape[0]:
            raise ValueError("pool_mlp_backward_dx: cols must be in [1, %d] (the rows of Wm), got %d" % (W.shape[0], cols))
        nbytes = lib().gs_pool_mlp_dx_pack_bytes(cols, W.shape[1])
        if nbytes < 0:
            raise ValueError("pool_mlp_backward_dx: needs 1 <= cols and hidden %% 128 == 0 (cols=%d hidden=%d)"
                             % (cols, W.shape[1]))
        ws = torch.empty((nbytes,), dtype=torch.uint8, device=W.device)
        Wc = W.contiguous()
        check(lib().gs_pool_mlp_dx_pack(ptr(Wc), Wc.stride(0), cols, Wc.shape[1], ptr(ws), stream_ptr()))
        _launched(1)
        return ws


def pool_mlp_backward_dp(table, n_groups, k, W, bias, packed, dhp, row_ids=None, row0=0, K=None, pool="max"):
    """B1 of the pooling branch's backward (gs_pool_mlp_backward_dp): recomputes pre = X W of maxpool_mlp_fused's rows
    and returns a uint8 buffer with dP = bf16(dpre) as dP^T tile images, then the fp32 per-tile column sums of dpre
    (contract: include/graphsage_b200.h, oracle/pool_grad.py).  dhp: float32 [n_groups, hidden], unit column stride."""
    require_cuda(table, W, bias, row_ids, dhp)
    if table.dtype != torch.bfloat16 or table.stride(1) != 1:
        raise TypeError("table must be row-major bfloat16")
    K = _check_mlp_K(W, K)
    hidden = W.shape[1]
    if dhp.dtype != torch.float32 or dhp.dim() != 2 or dhp.stride(1) != 1 or tuple(dhp.shape) != (n_groups, hidden):
        raise ValueError("dhp must be a float32 [%d, %d] matrix with unit column stride" % (n_groups, hidden))
    nbytes = lib().gs_pool_mlp_dp_bytes(n_groups, k, hidden)
    if nbytes < 0:
        raise ValueError("pool_mlp_backward_dp: needs k <= 128 and hidden %% 128 == 0 (k=%d hidden=%d)" % (k, hidden))
    grad = torch.empty((max(nbytes, 16),), dtype=torch.uint8, device=table.device)
    if row_ids is not None:
        row_ids = _i32(row_ids.reshape(-1), "row_ids")
    ws = packed.get(W)
    ev = _probe("pool_mlp_backward_dp/%d" % n_groups)
    check(lib().gs_pool_mlp_backward_dp(ptr(table), table.shape[0], K, table.stride(0), ptr(row_ids), row0, n_groups, k,
                                        ptr(ws), ptr(bias), hidden, ptr(dhp), dhp.stride(0), int(pool == "mean"), ptr(grad),
                                        stream_ptr()))
    _launched(1 if n_groups else 0, ev)
    return grad


def pool_mlp_backward_dw(table, n_groups, k, grad, dWm, dbm, row_ids=None, row0=0, K=None):
    """B2 (gs_pool_mlp_backward_dw): dWm += X^T dP over the re-gathered rows and dbm += the column sums of dpre, both in
    a fixed order.  dWm: contiguous float32 [K, hidden]; dbm: float32 [hidden]; grad: pool_mlp_backward_dp's buffer."""
    require_cuda(table, grad, dWm, dbm, row_ids)
    K = dWm.shape[0] if K is None else K
    hidden = dWm.shape[1]
    if dWm.dtype != torch.float32 or not dWm.is_contiguous() or dbm.dtype != torch.float32 or not dbm.is_contiguous() \
            or dbm.numel() != hidden:
        raise ValueError("dWm must be a contiguous float32 [K, hidden] matrix and dbm a contiguous float32 [hidden]")
    nbytes = lib().gs_pool_mlp_dw_workspace_bytes(n_groups, k, K, hidden)
    if nbytes < 0:
        raise ValueError("pool_mlp_backward_dw: needs k <= 128 and hidden %% 128 == 0 (k=%d hidden=%d)" % (k, hidden))
    ws = torch.empty((max(nbytes, 16),), dtype=torch.uint8, device=table.device)
    if row_ids is not None:
        row_ids = _i32(row_ids.reshape(-1), "row_ids")
    ev = _probe("pool_mlp_backward_dw/%d" % n_groups)
    check(lib().gs_pool_mlp_backward_dw(ptr(table), table.shape[0], K, table.stride(0), ptr(row_ids), row0, n_groups, k,
                                        hidden, ptr(grad), ptr(ws), nbytes, ptr(dWm), dWm.stride(0), ptr(dbm), stream_ptr()))
    _launched(4 if n_groups else 0, ev)                 # the GEMM, then the dWm, dbm-group and dbm sums
    return dWm, dbm


def pool_mlp_backward_dx(grad, n_groups, k, W, packed_dx, out=None):
    """B3 (gs_pool_mlp_backward_dx): dx = (dP Wm^T)[:, :cols] for the n_groups * k gathered rows, float32
    [n_groups * k, cols] (cols = packed_dx.cols); packed_dx: a PackedMlpDxWeights."""
    require_cuda(grad, W, out)
    cols, hidden = packed_dx.cols, W.shape[1]
    if out is None:
        out = torch.empty((n_groups * k, pad_cols(cols)), dtype=torch.float32, device=grad.device)[:, :cols]
    if out.dtype != torch.float32 or out.stride(1) != 1 or out.shape[0] < n_groups * k or out.shape[1] < cols:
        raise ValueError("out must be a row-major float32 [>= %d, >= %d] matrix" % (n_groups * k, cols))
    ws = packed_dx.get(W)
    ev = _probe("pool_mlp_backward_dx/%d" % n_groups)
    check(lib().gs_pool_mlp_backward_dx(n_groups, k, hidden, ptr(grad), ptr(ws), cols, ptr(out), out.stride(0), stream_ptr()))
    _launched(1 if n_groups else 0, ev)
    return out


def dropout_site(site):
    """(seed, call, rate) or (seed, call, rate, call_dev) -> the C descriptor; rate must lie in [0, 1) (the mask contract
    is in the header and oracle/dropout.py).  call_dev: None, or an int64 CUDA tensor whose first element the kernel adds to
    `call` when it runs (a CUDA graph replays with whatever it holds then)."""
    seed, call, rate = site[:3]
    call_dev = site[3] if len(site) > 3 else None
    rate = float(rate)
    if not 0.0 <= rate < 1.0:
        raise ValueError("dropout rate must be in [0, 1) (got %r)" % (rate,))
    if call_dev is not None:
        require_cuda(call_dev)
        if call_dev.dtype != torch.int64 or call_dev.numel() < 1:
            raise TypeError("call_dev must be an int64 CUDA tensor with >= 1 element")
    return _lib.DropoutSite(int(seed) & _U64, int(call) & 0xFFFFFFFF, rate, ptr(call_dev))


def gather_mean_dropout(src, segments, neigh_sites, self_sites, include_self=False, want_self=True, out_pitch=None):
    """gather_mean with training dropout (gs_gather_mean_dropout; reference aggregators.py:46-47 / 104-105): every gathered
    neighbour row and self row is dropped in registers with its segment's site before the fanout mean.  neigh_sites /
    self_sites: one (seed, call, rate) per segment.  Returns (dropped self rows or None, out_mean), [rows, out_pitch]."""
    require_cuda(src)
    if hasattr(src, "c_table") or src.dtype != torch.float32 or src.dim() != 2 or src.stride(1) != 1:
        raise ValueError("gather_mean_dropout needs a row-major float32 CUDA table")
    if len(segments) > _lib.MAX_SEGMENTS or len(neigh_sites) != len(segments) or len(self_sites) != len(segments):
        raise ValueError("gather_mean_dropout takes at most %d segments and one neighbour and one self site per segment"
                         % _lib.MAX_SEGMENTS)
    F = src.shape[1]
    if out_pitch is None:
        out_pitch = pad_cols(F)
    rows = max([s.out_row0 + s.n for s in segments] + [0])
    out_mean = torch.empty((rows, out_pitch), dtype=torch.float32, device=src.device)
    out_self = torch.empty((rows, out_pitch), dtype=torch.float32, device=src.device) if want_self else None
    nseg = max(len(segments), 1)
    arr = (Segment * nseg)(*[s.c_struct() for s in segments])
    ns = (_lib.DropoutSite * nseg)(*[dropout_site(x) for x in neigh_sites])
    ss = (_lib.DropoutSite * nseg)(*[dropout_site(x) for x in self_sites])
    ev = _probe("gather_mean_dropout/%d" % rows)
    check(lib().gs_gather_mean_dropout(ptr(src), src.shape[0], F, src.stride(0), arr, len(segments), ns, ss,
                                       int(bool(include_self)), ptr(out_self), ptr(out_mean), out_pitch, stream_ptr()))
    _launched(1 if rows else 0, ev)
    return out_self, out_mean


def dropout_apply(x, site, rows=None, group=1, scale=1.0, out=None, accumulate=False, pos_ids=None):
    """Masked scale (gs_dropout_apply): out[r, c] (+)= keep(site, pos, c) ? (x[r // group, c] * scale) / keep : 0 for
    r < rows (default x.shape[0] * group), pos = pos_ids[r] (an int32 CUDA tensor of >= rows ids) or r.  x, out: float32
    CUDA matrices with unit column stride (strided rows are fine).  Forward dropout (x -> drop(x)) and every dropout
    backward (the same mask applied to the incoming gradient).  Returns out (a new [rows, F] tensor unless given)."""
    require_cuda(x, out, pos_ids)
    group = int(group)
    if group < 1:
        raise ValueError("group must be >= 1")
    if x.dtype != torch.float32 or x.dim() != 2 or (x.stride(1) != 1 and x.shape[1] > 1):
        raise ValueError("x must be a float32 matrix with unit column stride")
    F = x.shape[1]
    rows = x.shape[0] * group if rows is None else int(rows)
    if x.shape[0] < (rows + group - 1) // group:
        raise ValueError("x has %d rows, %d needed" % (x.shape[0], (rows + group - 1) // group))
    c_site = dropout_site(site)
    if out is None:
        if accumulate:
            raise ValueError("accumulate needs out")
        out = torch.empty((rows, F), dtype=torch.float32, device=x.device)
    if out.dtype != torch.float32 or out.dim() != 2 or out.shape[0] < rows or out.shape[1] != F \
            or (out.stride(1) != 1 and F > 1):
        raise ValueError("out must be a float32 [>= %d, %d] matrix with unit column stride" % (rows, F))
    ldx, ldo = max(x.stride(0), F), max(out.stride(0), F)
    if out.data_ptr() == x.data_ptr() and (group != 1 or ldx != ldo):
        raise ValueError("in-place dropout_apply needs group == 1 and equal row strides")
    if pos_ids is not None:
        pos_ids = _i32(pos_ids.reshape(-1), "pos_ids")
        if pos_ids.numel() < rows:
            raise ValueError("pos_ids has %d ids, %d rows" % (pos_ids.numel(), rows))
    ev = _probe("dropout_apply/%d" % rows)
    check(lib().gs_dropout_apply(ptr(x), ldx, rows, F, group, float(scale), c_site, int(bool(accumulate)), ptr(out), ldo,
                                 ptr(pos_ids), stream_ptr()))
    _launched(1 if rows * F else 0, ev)
    return out


def _embed_lists(lists, d, who):
    """(ids, grad, group, scale) tuples -> (gs_embed_grad_list array, the int32 id tensors kept alive, device)."""
    if len(lists) > _lib.MAX_EMBED_LISTS:
        raise ValueError("%s takes at most %d lists" % (who, _lib.MAX_EMBED_LISTS))
    arr = (_lib.EmbedGradList * max(len(lists), 1))()
    keep = []
    dev = None
    for i, (ids, grad, group, scale) in enumerate(lists):
        require_cuda(ids, grad)
        ids = _i32(ids.reshape(-1), "ids")
        n, group = ids.numel(), int(group)
        if group < 1:
            raise ValueError("group must be >= 1")
        if grad.dtype != torch.float32 or grad.dim() != 2 or (grad.stride(1) != 1 and grad.shape[1] > 1) \
                or grad.shape[1] < d or grad.shape[0] < (n + group - 1) // group:
            raise ValueError("list %d: grad must be a float32 [>= %d, >= %d] matrix with unit column stride"
                             % (i, (n + group - 1) // group, d))
        keep.append(ids)
        dev = grad.device
        arr[i] = _lib.EmbedGradList(ptr(ids), ptr(grad), max(grad.stride(0), d), n, group, float(scale))
    return arr, keep, dev


def embedding_grad(lists, n_rows, d, out=None, sites=None):
    """Dense gradient of the trainable embedding table (gs_embedding_grad; the densified IndexedSlices gradient of
    tf.nn.embedding_lookup at reference graphsage/models.py:299): out[r] = sum of scale * grad[i // group] over every
    (ids, grad, group, scale) list entry i with ids[i] == r.  grad: float32 CUDA [>= ceil(n / group), >= d] with unit
    column stride (a strided view is fine).  Returns out, a contiguous float32 [n_rows, d]; deterministic.
    sites: optional (seed, call, rate) per list (gs_embedding_grad_dropout): entry i of list l is masked with site l at
    position i, (scale * grad) / keep where kept, 0 where dropped - the gradient through training dropout."""
    if sites is not None and len(sites) != len(lists):
        raise ValueError("embedding_grad: one site per list")
    arr, keep, dev = _embed_lists(lists, d, "embedding_grad")
    if out is None:
        out = torch.empty((n_rows, d), dtype=torch.float32, device=dev if dev is not None else "cuda")
    require_cuda(out)
    if out.dtype != torch.float32 or out.dim() != 2 or out.shape[0] != n_rows or out.shape[1] != d \
            or (out.stride(1) != 1 and d > 1):
        raise ValueError("out must be a float32 [%d, %d] matrix with unit column stride" % (n_rows, d))
    nbytes = lib().gs_embedding_grad_workspace_bytes(arr, len(lists), int(n_rows), int(d))
    if nbytes < 0:
        check(-1)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=out.device) if nbytes > 0 else None
    ev = _probe("embedding_grad/%d" % sum(k.numel() for k in keep))
    if sites is None:
        check(lib().gs_embedding_grad(arr, len(lists), int(n_rows), int(d), ptr(out), max(out.stride(0), d), ptr(ws), nbytes,
                                      stream_ptr()))
    else:
        c_sites = (_lib.DropoutSite * max(len(sites), 1))(*[dropout_site(s) for s in sites])
        check(lib().gs_embedding_grad_dropout(arr, c_sites, len(lists), int(n_rows), int(d), ptr(out), max(out.stride(0), d),
                                              ptr(ws), nbytes, stream_ptr()))
    _launched(3 if nbytes > 0 and n_rows * d else 0, ev)           # keys, chunk sums, combine (+ CUB's sort passes)
    return out


def _fp32_table(t, name, min_cols):
    require_cuda(t)
    if t.dtype != torch.float32 or t.dim() != 2 or (t.stride(1) != 1 and t.shape[1] > 1) or t.shape[1] < min_cols:
        raise ValueError("%s must be a float32 CUDA matrix with >= %d columns and unit column stride" % (name, min_cols))


def embedding_sgd(table, lists, lr):
    """Sparse gradient-descent update (gs_embedding_sgd; tf.train.GradientDescentOptimizer on the IndexedSlices gradient of
    embedding_lookup, reference graphsage/models.py:476): table[r] += -lr * (sum of scale * grad[i // group] over every
    (ids, grad, group, scale) entry i with ids[i] == r), in place, for the touched rows only; duplicate ids - also across
    lists - are summed first, in the deterministic order of embedding_grad.  table: float32 CUDA [n_rows, d], unit column
    stride (a strided view, e.g. the embedding columns of a wider table, is fine).  Returns table."""
    _fp32_table(table, "table", 1)
    n_rows, d = table.shape
    arr, keep, _ = _embed_lists(lists, d, "embedding_sgd")
    nbytes = lib().gs_embedding_grad_workspace_bytes(arr, len(lists), int(n_rows), int(d))
    if nbytes < 0:
        check(-1)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=table.device) if nbytes > 0 else None
    ev = _probe("embedding_sgd/%d" % sum(k.numel() for k in keep))
    check(lib().gs_embedding_sgd(arr, len(lists), int(n_rows), int(d), -float(lr), ptr(table), max(table.stride(0), d), ptr(ws),
                                 nbytes, stream_ptr()))
    _launched(3 if nbytes > 0 and n_rows * d else 0, ev)           # keys, chunk sums, combine (+ CUB's sort passes)
    return table


def skipgram_grad(target, context, batch1, batch2, neg):
    """One skip-gram forward + backward of Node2VecModel (gs_skipgram_grad; reference graphsage/models.py:459-501).
    target: float32 CUDA [V, d]; context: float32 CUDA [V, d + 1], its column d the context bias (unit column strides,
    strided rows fine).  batch1 / batch2: the B pairs, neg: the S shared negatives (int32 ids).  Returns a dict of new
    tensors: loss (0-d), aff [B] and neg_aff [B, S] (without the biases), gt [B, d] (gradient of target[batch1]),
    gc_pos [B, d + 1] and gc_neg [S, d + 1] (gradients of the context rows, bias gradient in column d).  Deterministic."""
    _fp32_table(target, "target", 1)
    d = target.shape[1]
    _fp32_table(context, "context", d + 1)
    if context.shape[0] != target.shape[0]:
        raise ValueError("target and context must have the same number of rows")
    require_cuda(batch1, batch2, neg)
    batch1, batch2, neg = _i32(batch1.reshape(-1), "batch1"), _i32(batch2.reshape(-1), "batch2"), _i32(neg.reshape(-1), "neg")
    B, S = batch1.numel(), neg.numel()
    if batch2.numel() != B or B < 1:
        raise ValueError("batch1 and batch2 must hold the same number (>= 1) of ids")
    if not 1 <= S <= _lib.MAX_UNIQUE_SAMPLED:
        raise ValueError("the number of negatives must be in [1, %d] (got %d)" % (_lib.MAX_UNIQUE_SAMPLED, S))
    dev = target.device
    f32 = dict(dtype=torch.float32, device=dev)
    wd = pad_cols(d + 1)
    out = dict(loss=torch.empty((), **f32), aff=torch.empty((B,), **f32), neg_aff=torch.empty((B, S), **f32),
               gt=torch.empty((B, pad_cols(d)), **f32)[:, :d], gc_pos=torch.empty((B, wd), **f32)[:, :d + 1],
               gc_neg=torch.empty((S, wd), **f32)[:, :d + 1])
    nbytes = lib().gs_skipgram_workspace_bytes(B, S, d)
    if nbytes < 0:
        check(-1)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
    ev = _probe("skipgram_grad/%d" % B)
    check(lib().gs_skipgram_grad(ptr(target), target.stride(0), ptr(context), context.stride(0), target.shape[0], d, ptr(batch1),
                                 ptr(batch2), B, ptr(neg), S, ptr(out["loss"]), ptr(out["aff"]), ptr(out["neg_aff"]),
                                 ptr(out["gt"]), out["gt"].stride(0), ptr(out["gc_pos"]), ptr(out["gc_neg"]), wd, ptr(ws), nbytes,
                                 stream_ptr()))
    _launched(2, ev)
    return out


def _rows_f32(t, name, cols):
    require_cuda(t)
    if t.dtype != torch.float32 or t.dim() != 2 or t.stride(1) != 1 or t.shape[1] < cols:
        raise ValueError("%s must be a row-major float32 matrix with >= %d columns" % (name, cols))
    return t


def seq_lengths(x, n, k):
    """The reference's sequence lengths (aggregators.py:411-414) of n sequences of k rows of x [n*k, K]: int32 [n],
    max(1, number of rows with an element that is not zero)."""
    _rows_f32(x, "x", 0)
    if x.shape[0] != n * k:
        raise ValueError("x has %d rows, expected n*k = %d" % (x.shape[0], n * k))
    out = torch.empty((n,), dtype=torch.int32, device=x.device)
    ev = _probe("seq_lengths/%d" % n)
    check(lib().gs_seq_lengths(ptr(x), x.stride(0), n, k, x.shape[1], ptr(out), stream_ptr()))
    _launched(1 if n else 0, ev)
    return out


def lstm_forward(P, Wh, lengths, n, k, out=None, train=False):
    """BasicLSTMCell under dynamic_rnn (aggregators.py:410-433): P [n*k, 4H] = X W_x + b, Wh [H, 4H] (a strided view is
    fine), lengths int32 [n].  Returns h_last [n, H] (into `out` when given); with train=True (h_last, gates [n*k, 4H],
    c [n*k, H], h_prev [n*k, H]) for lstm_backward and the weight gradients."""
    H = Wh.shape[0]
    _rows_f32(P, "P", 4 * H)
    _rows_f32(Wh, "Wh", 4 * H)
    lengths = _i32(lengths, "lengths")
    dev = P.device
    if out is None:
        out = torch.empty((n, H), dtype=torch.float32, device=dev)
    _rows_f32(out, "out", H)
    saved = [torch.empty((n * k, w), dtype=torch.float32, device=dev) for w in (4 * H, H, H)] if train else [None] * 3
    g, c, hp = saved
    ev = _probe("lstm_forward/%d" % n)
    check(lib().gs_lstm_forward(ptr(P), P.stride(0), ptr(Wh), Wh.stride(0), ptr(lengths), n, k, H, ptr(out), out.stride(0),
                                ptr(g), 4 * H, ptr(c), H, ptr(hp), H, stream_ptr()))
    _launched(1 if n else 0, ev)
    return (out, g, c, hp) if train else out


def lstm_backward(dh_last, gates, c, lengths, Wh, n, k):
    """Backpropagation through time of lstm_forward: dZ [n*k, 4H], the gradient of the gate pre-activations."""
    H = Wh.shape[0]
    _rows_f32(dh_last, "dh_last", H)
    _rows_f32(gates, "gates", 4 * H)
    _rows_f32(c, "c", H)
    _rows_f32(Wh, "Wh", 4 * H)
    lengths = _i32(lengths, "lengths")
    dz = torch.empty((n * k, 4 * H), dtype=torch.float32, device=gates.device)
    ev = _probe("lstm_backward/%d" % n)
    check(lib().gs_lstm_backward(ptr(dh_last), dh_last.stride(0), ptr(gates), gates.stride(0), ptr(c), c.stride(0),
                                 ptr(lengths), ptr(Wh), Wh.stride(0), n, k, H, ptr(dz), dz.stride(0), stream_ptr()))
    _launched(1 if n else 0, ev)
    return dz


def l2_normalize_rows_(x):
    """In-place tf.nn.l2_normalize(x, 1) - reference graphsage/models.py:368."""
    require_cuda(x)
    check(lib().gs_l2_normalize_rows(ptr(x), x.shape[0], x.shape[1], x.stride(0), stream_ptr()))
    _launched(1 if x.numel() else 0)
    return x
