"""Minibatches over sampled neighbourhoods: the contract of gs_csr_sampled_blocks (ops.csr_blocks with fanouts), of
gs_csr_sample_rows (ops.sample_csr_rows) and of the sampled_minibatch_* methods.  Plain numpy, in the kernels' order.

The sample S_l(v) of node v < N (the dummy node is N) at layer l, from its raw CSR row of d entries, fanout k = k_l:
  d <= k   every entry, in CSR order;
  d >  k   k distinct entry POSITIONS by Floyd's algorithm: for i = 0 .. k-1, j = d - k + i, t = (u_i * (j + 1)) >> 32;
           take t unless it is already taken, else take j.  The k positions are then sorted ascending, so a row of S_l
           keeps CSR order.
Entries are positions, not ids: an id repeated in a row can be drawn twice, as two entries.  An entry outside [0, N) is
read as N where the blocks read it (full_neighbor_blocks.clamp_ids); an empty row stays empty, and the block reads the
dummy for it, as the whole-neighbourhood blocks do.
u_i = word 0 of philox4x32_10(counter = (i, v, call mod 2^32, STREAM_SAMPLED_BLOCKS | l), key = split64(seed)).  The
stream [0x70000000, 0x70000008) lies past every other stream's word-3 range.
Rounding bias: t = floor(u (j + 1) / 2^32), u uniform on [0, 2^32), takes each value of [0, j] for floor or ceil of
2^32 / (j + 1) words, so each probability is within 2^-32 of 1 / (j + 1) and a step's law is biased by at most j / 2^32
(L1 distance to uniform on [0, j]).  Floyd's algorithm is exact (every k-subset equally likely) up to that bias.
1 <= k <= 256 (MAX_FANOUT); anything else is a ValueError.

Blocks: S_l over all nodes is a CSR (sample_rows), and block l is exactly oracle/full_neighbor_blocks.py's block built
over S_l: V_l = sorted-unique(V_{l+1}  u  the clamped entries of S_l over V_{l+1}'s nodes  u  {N}), with the same
src_ids / indptr / indices / rows layout.  So every bit-for-bit argument of that module holds for block l over S_l:
the layer computes, for V_{l+1}'s nodes, the whole-graph layer over S_l.  Block l uses fanouts[l]; for a model,
fanouts[l] = layer_infos[l].num_samples, so block L-1 (hop 1 from the seeds) uses layer_infos[L-1], as the reference's
sample() pairs hops with layer_infos.  A model's (seed, call) are its neigh_sampler's (seed, counter); one block set
advances the counter by exactly 1.

Test infrastructure - not imported by the product.
"""
import numpy as np

from .aggregate import l2_normalize, relu
from .full_neighbor import layer
from .full_neighbor_blocks import clamp_ids, csr_blocks
from .full_neighbor_grad import _layer_backward, _layer_forward, scatter_rows
from .numerics import gather_clamped
from .philox import philox4x32_10, split64

STREAM_SAMPLED_BLOCKS = 0x70000000
MAX_FANOUT = 256
MAX_LAYERS = 8


def check_fanout(k):
    k = int(k)
    if not 1 <= k <= MAX_FANOUT:
        raise ValueError("a fanout must be in [1, %d] (got %d)" % (MAX_FANOUT, k))
    return k


def draws(nodes, k, seed, call, layer):
    """uint32 [len(nodes), k]: u_i of each node."""
    nodes = np.asarray(nodes, dtype=np.int64).reshape(-1)
    ctr = np.empty((len(nodes), k, 4), dtype=np.uint32)
    ctr[..., 0] = np.arange(k, dtype=np.uint32)[None, :]
    ctr[..., 1] = nodes.astype(np.uint32)[:, None]
    ctr[..., 2] = np.uint32(int(call) & 0xFFFFFFFF)
    ctr[..., 3] = np.uint32(STREAM_SAMPLED_BLOCKS | int(layer))
    return philox4x32_10(ctr, np.array(split64(seed), dtype=np.uint32))[..., 0]


def floyd_positions(u, d):
    """int64 [n, k]: Floyd's positions, in draw order, for rows of lengths d (all > k) from their draws u [n, k]."""
    u = np.asarray(u, dtype=np.uint64)
    d = np.asarray(d, dtype=np.int64)
    n, k = u.shape
    held = np.full((n, k), -1, dtype=np.int64)
    for i in range(k):
        j = d - k + i
        t = ((u[:, i] * (j + 1).astype(np.uint64)) >> np.uint64(32)).astype(np.int64)
        taken = (held[:, :i] == t[:, None]).any(axis=1)
        held[:, i] = np.where(taken, j, t)
    return held


def sample_rows(indptr, indices, k, seed, call, layer, nodes=None):
    """S_layer as a CSR over all N nodes: (indptr int64 [N + 1], indices int64), entries as stored (not clamped) - what
    ops.sample_csr_rows returns.  nodes: sample only these rows (the others are left empty), as the blocks do."""
    k = check_fanout(k)
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int64)
    N = len(indptr) - 1
    lo = indptr[:-1]
    deg = np.maximum(indptr[1:] - lo, 0)
    if nodes is not None:
        keep = np.zeros(N, bool)
        nodes = np.asarray(nodes, dtype=np.int64).reshape(-1)
        keep[nodes[(nodes >= 0) & (nodes < N)]] = True
        deg = np.where(keep, deg, 0)
    cnt = np.minimum(deg, k)
    out_ptr = np.zeros(N + 1, dtype=np.int64)
    out_ptr[1:] = np.cumsum(cnt)
    out = np.empty(int(out_ptr[-1]), dtype=np.int64)
    short = np.nonzero((deg > 0) & (deg <= k))[0]
    if len(short):
        seg = np.repeat(np.arange(len(short)), deg[short])
        first = np.repeat(np.cumsum(deg[short]) - deg[short], deg[short])
        off = np.arange(len(seg), dtype=np.int64) - first
        out[out_ptr[short][seg] + off] = indices[lo[short][seg] + off]
    hub = np.nonzero(deg > k)[0]
    if len(hub):
        pos = np.sort(floyd_positions(draws(hub, k, seed, call, layer), deg[hub]), axis=1)
        out[(out_ptr[hub][:, None] + np.arange(k)[None, :]).reshape(-1)] = indices[(lo[hub][:, None] + pos).reshape(-1)]
    return out_ptr, out


def sampled_blocks(indptr, indices, seeds, fanouts, seed, call):
    """The L = len(fanouts) blocks over the samples: a list, index l = layer l, of full_neighbor_blocks.csr_blocks'
    dicts {src_ids, indptr, indices, rows}, block l built over S_l (fanout fanouts[l])."""
    fanouts = [check_fanout(k) for k in fanouts]
    if not 1 <= len(fanouts) <= MAX_LAYERS:
        raise ValueError("n_layers must be in [1, %d]" % MAX_LAYERS)
    N = len(indptr) - 1
    L = len(fanouts)
    blocks = [None] * L
    nxt = clamp_ids(seeds, N)
    for l in range(L - 1, -1, -1):
        s_ptr, s_idx = sample_rows(indptr, indices, fanouts[l], seed, call, l, nodes=np.unique(nxt))
        blocks[l] = csr_blocks(s_ptr, s_idx, nxt, 1)[0]
        nxt = blocks[l]["src_ids"].astype(np.int64)
    return blocks


def sampled_embeddings(features, indptr, indices, aggregators, concat, seeds, fanouts, seed, call, normalize=True):
    """The sampled_minibatch_embeddings of seeds: every layer over its sampled block, layer 0 on V_0's gathered rows
    through block 0.  float32 [len(seeds), w]."""
    features = np.asarray(features, dtype=np.float32)
    L = len(aggregators)
    blocks = sampled_blocks(indptr, indices, seeds, fanouts, seed, call)
    h = gather_clamped(features, blocks[0]["src_ids"])
    for l, agg in enumerate(aggregators):
        b = blocks[l]
        h = layer(agg, h, b["indptr"], b["indices"], b["rows"], concat, (lambda x: x) if l == L - 1 else relu)
    return l2_normalize(h) if normalize else h


def sampled_loss_grads(features, indptr, indices, aggregators, concat, node_ids, labels, pred_weights, pred_bias,
                       fanouts, seed, call, sigmoid_loss=False, weight_decay=0.0, identity_dim=0):
    """oracle.full_neighbor_blocks.block_loss_grads over the sampled blocks: (loss, per-layer grads, head grads,
    d(embeddings) [N+1, d] or None), every layer in its block's local space."""
    features = np.asarray(features, dtype=np.float32)
    labels = np.asarray(labels, dtype=np.float64)
    L = len(aggregators)
    blocks = sampled_blocks(indptr, indices, node_ids, fanouts, seed, call)
    h = gather_clamped(features, blocks[0]["src_ids"])
    caches = []
    for l, agg in enumerate(aggregators):
        b = blocks[l]
        c = _layer_forward(agg, h, b["indptr"], b["indices"], b["rows"], concat, l == L - 1)
        caches.append(c)
        h = c["y"]
    out = l2_normalize(h).astype(np.float64)
    logits = out @ pred_weights + pred_bias
    n = logits.shape[0]
    if sigmoid_loss:
        loss = np.mean(np.maximum(logits, 0) - logits * labels + np.log1p(np.exp(-np.abs(logits))))
        dlog = (1.0 / (1.0 + np.exp(-logits)) - labels) / logits.size
    else:
        sh = logits - logits.max(axis=1, keepdims=True)
        logp = sh - np.log(np.exp(sh).sum(axis=1, keepdims=True))
        loss = np.mean(-(labels * logp).sum(axis=1))
        dlog = (np.exp(logp) * labels.sum(axis=1, keepdims=True) - labels) / n
    head = {"weights": out.T @ dlog + weight_decay * pred_weights, "bias": dlog.sum(axis=0) + weight_decay * pred_bias}
    loss += 0.5 * weight_decay * sum(float((np.asarray(v, np.float64) ** 2).sum()) for v in (pred_weights, pred_bias))
    dout = dlog @ np.asarray(pred_weights, np.float64).T
    y64 = h.astype(np.float64)
    nrm = np.sqrt(np.maximum((y64 * y64).sum(axis=1, keepdims=True), 1e-12))
    dy = (dout / nrm - y64 * ((dout * y64).sum(axis=1, keepdims=True)) / nrm ** 3).astype(np.float32)
    grads, demb = [None] * L, None
    for l in range(L - 1, -1, -1):
        agg, b = aggregators[l], blocks[l]
        g, dsrc = _layer_backward(agg, caches[l], dy, b["indptr"], b["indices"], b["rows"], concat, l == L - 1,
                                  l > 0 or identity_dim > 0)
        for k in g:
            if weight_decay and k not in ("mlp_weights", "mlp_bias"):
                g[k] = g[k] + weight_decay * agg[k]
                loss += 0.5 * weight_decay * float((np.asarray(agg[k], np.float64) ** 2).sum())
        grads[l] = g
        if l > 0:
            dy = dsrc.astype(np.float32)
        elif identity_dim > 0:
            demb = scatter_rows(dsrc[:, :identity_dim], b["src_ids"], features.shape[0])
    return float(loss), grads, head, demb
