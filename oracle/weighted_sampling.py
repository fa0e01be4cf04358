"""Sampling neighbours in proportion to edge weight: the contract of gs_csr_weighted_blocks_plan / _fill / _fill_offsets
(ops.csr_blocks(..., sample_weights=w)), gs_csr_sample_rows_weighted (ops.sample_csr_rows(..., weights=w)) and the
sample_weight= keyword of the sampled_minibatch_* methods.  Plain numpy, in the kernels' order, bit for bit.

sample_weight w is float32, one value per entry of `indices`, aligned with it.  It is data: no gradient flows to it.  It
is independent of edge_weight (oracle/weighted.py), and the two may be the same array.

The sample S_l^w(v) of node v < N at layer l with fanout k = k_l, from its raw CSR row of d entries:
  eligible   the entries with w_j > 0 (a NaN, zero or negative weight is never drawn); d+ = their number;
  d+ <= k    every eligible entry, in CSR order (d+ = 0: the row is empty, and the block reads the dummy for it, as it
             does for an empty raw row);
  d+ >  k    the k eligible entries with the smallest (key_j, j), compared lexicographically - position breaks ties -
             written in ascending position order, as the uniform sample is.
The key is the exponential race (Efraimidis & Spirakis): key_j = fl64(E_j / fl64(w_j)), E_j = neg_log(U_j),
U_j = (2m + 1) 2^-53 exactly, m = (a << 20) | (b >> 12), 52 bits from two Philox words (a, b) = words (0, 1) for even j,
(2, 3) for odd j of philox4x32_10(counter = (j >> 1, v, call mod 2^32, STREAM_WEIGHTED_BLOCKS | l), key = split64(seed)),
so one Philox call serves two entries.  STREAM_WEIGHTED_BLOCKS = 0x80000000: word 3 lies in [0x80000000, 0x80000008),
past every other stream (the highest, the uniform blocks', is [0x70000000, 0x70000008)).
A +inf weight gives key 0 and a subnormal weight may give key +inf; both are ordered by position among equal keys.
Keys are >= 0 (E >= 1.1e-16 > 0), so the kernels compare their bit patterns as unsigned integers.

The law.  With exact arithmetic E_j are independent Exp(1) and E_j / w_j ~ Exp(w_j): the entry with the smallest key is
entry j with probability w_j / sum(w), and, by memorylessness, the order of the smallest keys is successive sampling
without replacement in proportion to w.  So S^w is the set of the first k draws of that scheme.
Bias.  U takes the 2^52 midpoints of a grid of step 2^-52 on (0, 1), each with probability 2^-52 up to the Philox
words' own quality; the distribution function of U is within 2^-53 of the uniform one at every point, so each E_j is
within 2^-53 in Kolmogorov distance of Exp(1), and the law of the sample - a function of the d+ keys - is within
d+ 2^-53 (total variation) of the exact one from U alone.  neg_log is within 2 ulp of -ln U over every U this rule
makes (tests/test_weighted_sampling_cpu.py checks 2 ulp at the ends, at powers of two and at 10^6 random points) and is
monotone non-increasing in U, so it maps the grid order-preservingly; a relative error of 2^-51 moves each key by at
most that relative amount, which changes the selected set only where two keys lie within 2^-51 relatively, an event of
probability below d+^2 2^-50 per row.  The division E / w is correctly rounded, exact in its order up to such ties.
One block set advances the sampler's counter by exactly 1, as the uniform blocks do: block l draws with (call, l).

Blocks: block l is oracle/full_neighbor_blocks.py's csr_blocks over S_l^w (sample_rows over V_{l+1}), exactly as
oracle/sampled_blocks.py builds the uniform blocks over S_l; an entry's offset is its position in the raw row (the
held key's j), which training dropout and edge_weight read (oracle/sampled_blocks_dropout.py, oracle/weighted.py).

Test infrastructure - not imported by the product.
"""
import numpy as np

from . import weighted as wt
from .aggregate import l2_normalize
from .full_neighbor_blocks import clamp_ids, csr_blocks
from .full_neighbor_grad import scatter_rows
from .numerics import gather_clamped
from .philox import philox4x32_10, split64
from .sampled_blocks import MAX_LAYERS, check_fanout

STREAM_WEIGHTED_BLOCKS = 0x80000000

SQRT2 = float.fromhex("0x1.6a09e667f3bcdp+0")     # fl(sqrt(2))
LN2_HI = float.fromhex("0x1.62e42fee00000p-1")    # ln 2 = LN2_HI + LN2_LO; e * LN2_HI is exact for |e| < 2^21
LN2_LO = float.fromhex("0x1.a39ef35793c76p-33")
# the atanh series' coefficients 1 / (2n + 1), n = 1 .. 10, each correctly rounded to fp64
COEFFS = tuple(1.0 / (2 * n + 1) for n in range(1, 11))


def neg_log(u):
    """-ln(u) for fp64 u in (0, 1) normal, by a fixed sequence of IEEE fp64 operations (no FMA, no library log):
      u = f0 2^e0, f0 in [1, 2) (exact bit split);  f = f0 / 2, e = e0 + 1 when f0 > SQRT2, else f = f0, e = e0
      s = (f - 1) / (f + 1);  z = s * s;  P = c10;  P = P * z + c_n for n = 9 .. 1 (Horner)
      t = s + s;  lnf = t + t * (z * P)                                  (ln f = 2 atanh(s), |s| <= 0.1716)
      E = -((e * LN2_HI) + ((e * LN2_LO) + lnf))
    The kernels run the same sequence with __dadd_rn / __dmul_rn / __ddiv_rn, which are never contracted."""
    u = np.asarray(u, dtype=np.float64)
    bits = u.view(np.uint64)
    e0 = ((bits >> np.uint64(52)) & np.uint64(0x7FF)).astype(np.int64) - 1023
    f0 = ((bits & np.uint64(0x000FFFFFFFFFFFFF)) | np.uint64(0x3FF0000000000000)).view(np.float64)
    big = f0 > SQRT2
    f = np.where(big, f0 * 0.5, f0)
    e = (e0 + big).astype(np.float64)
    s = (f - 1.0) / (f + 1.0)
    z = s * s
    p = np.full_like(z, COEFFS[-1])
    for c in COEFFS[-2::-1]:
        p = p * z + c
    t = s + s
    lnf = t + t * (z * p)
    return -((e * LN2_HI) + ((e * LN2_LO) + lnf))


def uniforms(nodes, j, seed, call, layer):
    """fp64 U_j of entries j (raw-row positions) of nodes (same shape, broadcast): (2m + 1) 2^-53."""
    nodes, j = np.broadcast_arrays(np.asarray(nodes, dtype=np.int64), np.asarray(j, dtype=np.int64))
    ctr = np.empty(nodes.shape + (4,), dtype=np.uint32)
    ctr[..., 0] = (j >> 1).astype(np.uint32)
    ctr[..., 1] = nodes.astype(np.uint32)
    ctr[..., 2] = np.uint32(int(call) & 0xFFFFFFFF)
    ctr[..., 3] = np.uint32(STREAM_WEIGHTED_BLOCKS | int(layer))
    r = philox4x32_10(ctr, np.array(split64(seed), dtype=np.uint32)).astype(np.uint64)
    odd = (j & 1).astype(bool)
    a = np.where(odd, r[..., 2], r[..., 0])
    b = np.where(odd, r[..., 3], r[..., 1])
    m = (a << np.uint64(20)) | (b >> np.uint64(12))
    return (2 * m + 1).astype(np.float64) * 2.0 ** -53


def keys(nodes, j, w, seed, call, layer):
    """fp64 key_j = E_j / w_j of entries j of nodes with weights w (fp32, widened exactly)."""
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        return neg_log(uniforms(nodes, j, seed, call, layer)) / np.asarray(w, dtype=np.float32).astype(np.float64)


def sample_offsets(indptr, w, k, seed, call, layer, nodes=None):
    """S_layer^w as a CSR of raw-row offsets over all N nodes: (indptr int64 [N + 1], offsets int64), row v holding the
    ascending positions of its sample.  nodes: sample only these rows (the others are left empty), as the blocks do."""
    k = check_fanout(k)
    indptr = np.asarray(indptr, dtype=np.int64)
    N = len(indptr) - 1
    w = np.asarray(w)
    if w.dtype != np.float32 or w.ndim != 1:
        raise ValueError("sample weights must be a 1-D float32 array, one value per CSR entry")
    lo = indptr[:-1]
    deg = np.maximum(indptr[1:] - lo, 0)
    if nodes is not None:
        keep = np.zeros(N, bool)
        nodes = np.asarray(nodes, dtype=np.int64).reshape(-1)
        keep[nodes[(nodes >= 0) & (nodes < N)]] = True
        deg = np.where(keep, deg, 0)
    rows = np.nonzero(deg > 0)[0]
    seg = np.repeat(rows, deg[rows])                              # the node of every candidate entry
    first = np.repeat(np.cumsum(deg[rows]) - deg[rows], deg[rows])
    j = np.arange(len(seg), dtype=np.int64) - first               # its raw-row position
    wj = w[lo[seg] + j] if len(seg) else np.zeros(0, np.float32)
    with np.errstate(invalid="ignore"):
        ok = wj > 0
    seg, j, wj = seg[ok], j[ok], wj[ok]
    key = keys(seg, j, wj, seed, call, layer)
    order = np.lexsort((j, key.view(np.uint64), seg))             # by node, then (key, j)
    seg, j = seg[order], j[order]
    start = np.searchsorted(seg, seg, side="left")
    take = (np.arange(len(seg)) - start) < k                      # the k smallest (key, j) of each node
    seg, j = seg[take], j[take]
    order = np.lexsort((j, seg))                                  # ascending position within each node
    seg, j = seg[order], j[order]
    cnt = np.bincount(seg, minlength=N)[:N] if N else np.zeros(0, np.int64)
    out_ptr = np.zeros(N + 1, dtype=np.int64)
    out_ptr[1:] = np.cumsum(cnt)
    return out_ptr, j


def sample_rows(indptr, indices, w, k, seed, call, layer, nodes=None):
    """S_layer^w as a CSR over all N nodes: (indptr int64 [N + 1], indices int64), entries as stored (not clamped) -
    what ops.sample_csr_rows(..., weights=w) returns."""
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int64)
    out_ptr, off = sample_offsets(indptr, w, k, seed, call, layer, nodes)
    node = np.repeat(np.arange(len(out_ptr) - 1), np.diff(out_ptr))
    return out_ptr, indices[indptr[node] + off] if len(off) else np.zeros(0, np.int64)


def entry_offsets(indptr, indices, w, seeds, fanouts, seed, call):
    """(blocks, offsets): the L = len(fanouts) blocks over S_l^w - a list, index l = layer l, of
    full_neighbor_blocks.csr_blocks' dicts {src_ids, indptr, indices, rows} - and per block int64 [entries] aligned
    with its indices, each entry's raw-row offset: what ops.csr_blocks(..., sample_weights=w, entry_offsets=True)
    returns (offsets as int32)."""
    fanouts = [check_fanout(k) for k in fanouts]
    if not 1 <= len(fanouts) <= MAX_LAYERS:
        raise ValueError("n_layers must be in [1, %d]" % MAX_LAYERS)
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int64)
    N = len(indptr) - 1
    L = len(fanouts)
    blocks, offsets = [None] * L, [None] * L
    nxt = clamp_ids(seeds, N)
    for l in range(L - 1, -1, -1):
        o_ptr, o = sample_offsets(indptr, w, fanouts[l], seed, call, l, nodes=np.unique(nxt))
        node = np.repeat(np.arange(N), np.diff(o_ptr))
        s_idx = indices[indptr[node] + o] if len(o) else np.zeros(0, np.int64)
        b = blocks[l] = csr_blocks(o_ptr, s_idx, nxt, 1)[0]
        # a member row u of the block is S_l^w(src_ids[u]), in the same order: its offsets are that row of o
        cnt = np.diff(b["indptr"])
        v = np.asarray(b["src_ids"], dtype=np.int64)[:-1][cnt > 0]
        offsets[l] = (np.concatenate([o[o_ptr[x]:o_ptr[x + 1]] for x in v]) if len(v) else np.zeros(0, np.int64))
        nxt = b["src_ids"].astype(np.int64)
    return blocks, offsets


def sampled_blocks(indptr, indices, w, seeds, fanouts, seed, call):
    """The blocks of entry_offsets, without the offsets: what ops.csr_blocks(..., sample_weights=w) returns."""
    return entry_offsets(indptr, indices, w, seeds, fanouts, seed, call)[0]


def blocks_and_maps(indptr, indices, w, seeds, fanouts, seed, call):
    """(blocks, position maps) as oracle/sampled_blocks_dropout._blocks_and_maps builds them for the uniform blocks: the
    masks of a weighted sampled block name each entry by its raw CSR position, so the dropout rules hold unchanged."""
    blocks, offsets = entry_offsets(indptr, indices, w, seeds, fanouts, seed, call)
    return blocks, [(indptr, b["src_ids"], len(indices), o) for b, o in zip(blocks, offsets)]


def layer_graphs(indptr, indices, edge_weight, sample_weight, node_ids, fanouts, seed, call):
    """(V_0, [(graph, rows, src_ids)] per layer) over the weighted sampled blocks, as oracle/weighted.layer_graphs gives
    them for mode "sampled": each block entry carries its raw entry's edge weight (all ones when edge_weight is None)."""
    N = len(indptr) - 1
    ew = wt._weights(edge_weight, len(np.asarray(indices)))
    blocks, offs = entry_offsets(indptr, indices, sample_weight, clamp_ids(node_ids, N), fanouts, seed, call)
    out = [((b["indptr"], b["indices"], wt.block_weights(indptr, ew, b, o)), b["rows"], b["src_ids"])
           for b, o in zip(blocks, offs)]
    return blocks[0]["src_ids"], out


def embeddings(features, indptr, indices, sample_weight, aggregators, concat, node_ids, fanouts, seed, call,
               normalize=True, edge_weight=None):
    """sampled_minibatch_embeddings(..., sample_weight=, edge_weight=): float32 [len(node_ids), w]."""
    h = np.asarray(features, dtype=np.float32)
    v0, graphs = layer_graphs(indptr, indices, edge_weight, sample_weight, node_ids, fanouts, seed, call)
    h = gather_clamped(h, v0)
    L = len(aggregators)
    for l, (agg, (graph, rows, _)) in enumerate(zip(aggregators, graphs)):
        h = wt._layer_forward(agg, h, graph, rows, concat, l == L - 1)["y"]
    return l2_normalize(h) if normalize else h


def loss_grads(features, indptr, indices, sample_weight, aggregators, concat, node_ids, labels, pred_weights,
               pred_bias, fanouts, seed, call, sigmoid_loss=False, weight_decay=0.0, identity_dim=0, edge_weight=None):
    """The supervised step over the weighted sampled blocks (oracle/weighted.loss_grads' returns: loss, per-layer grads,
    head grads, d(embeddings) [N+1, d] or None)."""
    h = np.asarray(features, dtype=np.float32)
    labels = np.asarray(labels, dtype=np.float64)
    L = len(aggregators)
    v0, graphs = layer_graphs(indptr, indices, edge_weight, sample_weight, node_ids, fanouts, seed, call)
    h = gather_clamped(h, v0)
    caches = []
    for l, (agg, (graph, rows, _)) in enumerate(zip(aggregators, graphs)):
        caches.append(wt._layer_forward(agg, h, graph, rows, concat, l == L - 1))
        h = caches[-1]["y"]
    out = l2_normalize(h).astype(np.float64)
    logits = out @ pred_weights + pred_bias
    if sigmoid_loss:
        loss = np.mean(np.maximum(logits, 0) - logits * labels + np.log1p(np.exp(-np.abs(logits))))
        dlog = (1.0 / (1.0 + np.exp(-logits)) - labels) / logits.size
    else:
        sh = logits - logits.max(axis=1, keepdims=True)
        logp = sh - np.log(np.exp(sh).sum(axis=1, keepdims=True))
        loss = np.mean(-(labels * logp).sum(axis=1))
        dlog = (np.exp(logp) * labels.sum(axis=1, keepdims=True) - labels) / logits.shape[0]
    head = {"weights": out.T @ dlog + weight_decay * pred_weights, "bias": dlog.sum(axis=0) + weight_decay * pred_bias}
    loss += 0.5 * weight_decay * sum(float((np.asarray(v, np.float64) ** 2).sum()) for v in (pred_weights, pred_bias))
    dout = dlog @ np.asarray(pred_weights, np.float64).T
    y64 = h.astype(np.float64)
    nrm = np.sqrt(np.maximum((y64 * y64).sum(axis=1, keepdims=True), 1e-12))
    dy = (dout / nrm - y64 * ((dout * y64).sum(axis=1, keepdims=True)) / nrm ** 3).astype(np.float32)
    grads, demb = [None] * L, None
    for l in range(L - 1, -1, -1):
        agg, (graph, rows, src_ids) = aggregators[l], graphs[l]
        g, dsrc = wt._layer_backward(agg, caches[l], dy, graph, rows, concat, l == L - 1, l > 0 or identity_dim > 0)
        for key in g:
            if weight_decay and key not in ("mlp_weights", "mlp_bias"):
                g[key] = g[key] + weight_decay * agg[key]
                loss += 0.5 * weight_decay * float((np.asarray(agg[key], np.float64) ** 2).sum())
        grads[l] = g
        if l > 0:
            dy = dsrc.astype(np.float32)
        elif identity_dim > 0:
            demb = scatter_rows(dsrc[:, :identity_dim], src_ids, np.asarray(features).shape[0])
    return float(loss), grads, head, demb
