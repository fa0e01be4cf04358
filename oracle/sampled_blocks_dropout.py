"""Training dropout over sampled blocks: the contract of gs_csr_sampled_blocks_fill_offsets (ops.csr_blocks(...,
entry_offsets=True)), gs_csr_aggregate_dropout_offsets, ops.csr_slots_to_offsets and the `dropout=p` argument of the
sampled_minibatch_* training methods.  Plain numpy, fp32, in kernel order.

The masks are exactly those of oracle/full_neighbor_dropout.py - the same sites (full_neighbor_site_plan order, numbered
from the model's dropout_counter), counters and arithmetic, every position a GLOBAL identity.  One rule is new:
  neigh, sampled block   entry j of local row r of sampled block l has global node v = src_ids[r]; its position is
                         indptr[v] + q_j, q_j the entry's offset in v's raw CSR row: the (ascending) Floyd position when
                         d > k_l, j itself when d <= k_l (oracle/sampled_blocks.py's S_l(v)).
The implicit dummy entry of an empty row, of an out-of-range node and of the dummy node stays nnz + v; self, mlp and
head positions are unchanged (node ids; row r of node_ids for the head).  A sampled block 0's self rows are V_1's global
ids, which are their positions.
Consequences: a sampled entry is masked as the same edge is masked in the whole-graph pass, so the mask of a node's
layer-0 neighbour sum depends only on (site, node), not on the batch; and with every fanout >= the largest degree the
offsets are 0 .. d-1 and the blocks are csr_blocks' bytes, so the masked sampled minibatch equals the masked
whole-neighbourhood minibatch (full_neighbor_dropout.block_outputs) bit for bit.
Backward: the transposed sum masks by pos_indptr[g(i)] + t_slot; over a sampled block t_slot (the entry's slot in the
block row) is first mapped to the raw-row offset, t_slot' = offsets[block indptr[i] + t_slot] where t_slot >= 0, -1 and
-2 kept (slots_to_offsets).

Test infrastructure - not imported by the product.
"""
import numpy as np

from . import full_neighbor_dropout as fd
from .aggregate import l2_normalize, relu
from .dropout import apply as drop_rows
from .full_neighbor import _combine
from .full_neighbor_blocks import clamp_ids
from .full_neighbor_grad import mean_counts, scatter_rows
from .numerics import gather_clamped
from .sampled_blocks import check_fanout, draws, floyd_positions, sampled_blocks


def sample_offsets(indptr, k, seed, call, layer, nodes=None):
    """S_layer as a CSR of raw-row offsets over all N nodes: (indptr int64 [N + 1], offsets int64) - row v holds the
    offsets q of sample_rows' entries of v (0 .. d-1 when d <= k, else the sorted Floyd positions)."""
    k = check_fanout(k)
    indptr = np.asarray(indptr, dtype=np.int64)
    N = len(indptr) - 1
    deg = np.maximum(indptr[1:] - indptr[:-1], 0)
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
        out[out_ptr[short][seg] + off] = off
    hub = np.nonzero(deg > k)[0]
    if len(hub):
        pos = np.sort(floyd_positions(draws(hub, k, seed, call, layer), deg[hub]), axis=1)
        out[(out_ptr[hub][:, None] + np.arange(k)[None, :]).reshape(-1)] = pos.reshape(-1)
    return out_ptr, out


def entry_offsets(indptr, indices, seeds, fanouts, seed, call):
    """(blocks, offsets): sampled_blocks(...) and, per block, int64 [entries] aligned with its indices - what
    ops.csr_blocks(..., entry_offsets=True) returns (as int32)."""
    blocks = sampled_blocks(indptr, indices, seeds, fanouts, seed, call)
    offsets = []
    for l, b in enumerate(blocks):
        o_ptr, o = sample_offsets(indptr, fanouts[l], seed, call, l, nodes=b["src_ids"])
        cnt = np.diff(b["indptr"])
        rows = np.nonzero(cnt > 0)[0]
        v = b["src_ids"][rows].astype(np.int64)
        assert np.array_equal(cnt[rows], o_ptr[v + 1] - o_ptr[v])
        seg = np.repeat(np.arange(len(rows)), cnt[rows])
        first = np.repeat(np.cumsum(cnt[rows]) - cnt[rows], cnt[rows])
        offsets.append(o[o_ptr[v][seg] + np.arange(len(seg), dtype=np.int64) - first] if len(seg) else
                       np.zeros(0, np.int64))
    return blocks, offsets


def csr_aggregate_dropout_offsets(table, indptr, indices, op, neigh, self_site, pos_map, rows=None):
    """gs_csr_aggregate_dropout_offsets (ops "mean", "mean_self") bit for bit: fp32 [n, F].  pos_map = (pos_indptr,
    pos_ids or None, pos_nnz, pos_off): entry j of a row at lo is masked at pos_indptr[g] + pos_off[lo + j]."""
    table = np.asarray(table)
    R, F = table.shape
    indices = np.asarray(indices, dtype=np.int64)
    pos_off = np.asarray(pos_map[3], dtype=np.int64)
    nodes, lo, cnt, g, base = fd.row_bases(indptr, indices, rows, pos_map[:3], R)
    count = np.maximum(cnt, 1)
    acc = np.zeros((len(nodes), F), dtype=np.float32)
    for j in range(int(count.max()) if len(nodes) else 0):
        sel = np.nonzero(count > j)[0]
        ids = np.full(len(sel), R - 1, dtype=np.int64)
        pos = base[sel].copy()
        has = cnt[sel] > 0
        ids[has] = indices[lo[sel][has] + j]
        pos[has] += pos_off[lo[sel][has] + j]
        acc[sel] = acc[sel] + fd._drop(gather_clamped(table, ids), neigh, pos)
    if op == "mean_self":
        acc = acc + fd._drop(gather_clamped(table, nodes), self_site, g)
        return acc / (count + 1).astype(np.float32)[:, None]
    if op != "mean":
        raise ValueError(op)
    return acc / count.astype(np.float32)[:, None]


def slots_to_offsets(t_slot, t_indices, indptr, pos_off):
    """ops.csr_slots_to_offsets: t_slot >= 0 -> pos_off[indptr[t_indices] + t_slot]; -1 and -2 kept."""
    t_slot = np.asarray(t_slot, np.int64)
    i = np.asarray(t_indices, np.int64)
    pos_off = np.asarray(pos_off, np.int64)
    out = t_slot.copy()
    s = t_slot >= 0
    out[s] = pos_off[np.asarray(indptr, np.int64)[i[s]] + t_slot[s]]
    return out


def mean_backward_dropout_offsets(g, indptr, indices, with_self, neigh, self_site, pos_map):
    """d(src) of the masked mean over a sampled block's effective rows for the dense gradient g [N + 1, w]."""
    t_indptr, t_indices, t_slot = fd.csr_transpose_slots(indptr, indices, with_self)
    t_slot = slots_to_offsets(t_slot, t_indices, indptr, pos_map[3])
    gp = (np.asarray(g, dtype=np.float32) / mean_counts(indptr, with_self)[:, None]).astype(np.float32)
    return fd.csr_sum_dropout(gp, t_indptr, t_indices, t_slot, neigh, self_site, pos_map[:3])


def _layer_forward(agg, h, b, concat, last, s, pos_map):
    """One masked layer over sampled block b (h: the rows of b's src_ids), keeping what the backward reads."""
    if agg["type"] not in ("mean", "gcn"):         # the pools mask per node only: the whole-neighbourhood rule
        return fd._layer_forward(agg, h, b["indptr"], b["indices"], b["rows"], concat, last, s, pos_map[:3])
    c = {"h": h}
    if agg["type"] == "gcn":
        c["p"] = csr_aggregate_dropout_offsets(h, b["indptr"], b["indices"], "mean_self", s["neigh"], s["self"], pos_map,
                                               b["rows"])
        y = c["p"] @ agg["weights"]
    else:
        ids = fd.global_nodes(b["rows"], len(b["indptr"]) - 1, pos_map[1])
        c["hs"] = fd._drop(gather_clamped(h, b["rows"]), s["self"], ids)
        c["p"] = csr_aggregate_dropout_offsets(h, b["indptr"], b["indices"], "mean", s["neigh"], s["self"], pos_map,
                                               b["rows"])
        y = _combine(c["hs"] @ agg["self_weights"], c["p"] @ agg["neigh_weights"], concat)
    if agg.get("bias") is not None:
        y = y + agg["bias"]
    c["y"] = (y if last else relu(y)).astype(np.float32)
    return c


def _layer_backward(agg, c, dy, b, concat, last, need_dsrc, s, pos_map):
    """(weight gradients, d(layer input) [rows of src_ids, in] or None), every mask regenerated."""
    indptr, indices, rows = b["indptr"], b["indices"], b["rows"]
    if agg["type"] not in ("mean", "gcn"):
        return fd._layer_backward(agg, c, dy, indptr, indices, rows, concat, last, need_dsrc, s, pos_map[:3])
    n_rows = c["h"].shape[0]
    dz = dy if last else np.where(c["y"] > 0, dy, np.float32(0)).astype(np.float32)
    grads = {}
    if agg["type"] == "gcn":
        grads["weights"] = c["p"].T @ dz
        if not need_dsrc:
            return grads, None
        return grads, mean_backward_dropout_offsets(scatter_rows(dz @ agg["weights"].T, rows, n_rows), indptr, indices,
                                                    True, s["neigh"], s["self"], pos_map)
    D = agg["self_weights"].shape[1]
    dzs, dzn = (dz[:, :D], dz[:, D:]) if concat else (dz, dz)
    grads["self_weights"] = c["hs"].T @ dzs
    grads["neigh_weights"] = c["p"].T @ dzn
    if not need_dsrc:
        return grads, None
    dp = scatter_rows((dzn @ agg["neigh_weights"].T).astype(np.float32), rows, n_rows)
    node_mask = fd.global_nodes(np.arange(n_rows), len(indptr) - 1, pos_map[1])
    dself = fd._drop(scatter_rows(dzs @ agg["self_weights"].T, rows, n_rows), s["self"], node_mask)
    return grads, mean_backward_dropout_offsets(dp, indptr, indices, False, s["neigh"], s["self"], pos_map) + dself


def _blocks_and_maps(indptr, indices, seeds, fanouts, seed, call):
    blocks, offsets = entry_offsets(indptr, indices, seeds, fanouts, seed, call)
    maps = [(indptr, b["src_ids"], len(indices), o) for b, o in zip(blocks, offsets)]
    return blocks, maps


def sampled_block_outputs(features, indptr, indices, aggregators, concat, seeds, fanouts, seed, call, all_sites,
                          normalize=True):
    """The masked sampled_minibatch_outputs of seeds (no head): fp32 [len(seeds), w].  all_sites:
    full_neighbor_dropout.sites(kind, L, ...)."""
    features = np.asarray(features, dtype=np.float32)
    blocks, maps = _blocks_and_maps(indptr, indices, seeds, fanouts, seed, call)
    L = len(aggregators)
    h = gather_clamped(features, blocks[0]["src_ids"])
    for l, agg in enumerate(aggregators):
        h = _layer_forward(agg, h, blocks[l], concat, l == L - 1, fd._layer_sites(all_sites, l), maps[l])["y"]
    return l2_normalize(h) if normalize else h


def sampled_loss_grads_dropout(features, indptr, indices, aggregators, concat, node_ids, labels, pred_weights,
                               pred_bias, fanouts, seed, call, all_sites, sigmoid_loss=False, weight_decay=0.0,
                               identity_dim=0):
    """oracle.sampled_blocks.sampled_loss_grads with the masks of all_sites (sites(kind, L, True, ...)): the same
    returns (loss, per-layer grads, head grads, d(embeddings) [N+1, d] or None)."""
    features = np.asarray(features, dtype=np.float32)
    labels = np.asarray(labels, dtype=np.float64)
    node_ids = clamp_ids(node_ids, len(indptr) - 1)
    blocks, maps = _blocks_and_maps(indptr, indices, node_ids, fanouts, seed, call)
    L = len(aggregators)
    h = gather_clamped(features, blocks[0]["src_ids"])
    caches = []
    for l, agg in enumerate(aggregators):
        c = _layer_forward(agg, h, blocks[l], concat, l == L - 1, fd._layer_sites(all_sites, l), maps[l])
        caches.append(c)
        h = c["y"]
    head_site = all_sites[(None, "head")]
    out = drop_rows(l2_normalize(h), *head_site).astype(np.float64)
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
    dout = drop_rows((dlog @ np.asarray(pred_weights, np.float64).T).astype(np.float32), *head_site).astype(np.float64)
    y64 = h.astype(np.float64)
    nrm = np.sqrt(np.maximum((y64 * y64).sum(axis=1, keepdims=True), 1e-12))
    dy = (dout / nrm - y64 * ((dout * y64).sum(axis=1, keepdims=True)) / nrm ** 3).astype(np.float32)
    grads, demb = [None] * L, None
    for l in range(L - 1, -1, -1):
        agg = aggregators[l]
        g, dsrc = _layer_backward(agg, caches[l], dy, blocks[l], concat, l == L - 1, l > 0 or identity_dim > 0,
                                  fd._layer_sites(all_sites, l), maps[l])
        for k in g:
            if weight_decay and k not in ("mlp_weights", "mlp_bias"):
                g[k] = g[k] + weight_decay * agg[k]
                loss += 0.5 * weight_decay * float((np.asarray(agg[k], np.float64) ** 2).sum())
        grads[l] = g
        if l > 0:
            dy = dsrc.astype(np.float32)
        elif identity_dim > 0:
            demb = scatter_rows(dsrc[:, :identity_dim], blocks[0]["src_ids"], features.shape[0])
    return float(loss), grads, head, demb

