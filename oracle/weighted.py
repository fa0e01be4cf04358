"""Aggregation over weighted edges: the contract of gs_csr_aggregate_weighted, gs_csr_max_backward_weighted and the
edge_weight= keyword of the CSR-family entry points (full_neighbor_*, full_neighbor_minibatch_*, sampled_minibatch_*).
Plain numpy, fp32, in the kernels' order.

edge_weight w is float32, one value per entry of `indices`, aligned with it.  It is data, not a parameter: no gradient
flows to it.  Any finite value is allowed (zero, negative, large).  Message j of node v is fl(w_j * x_j): the product is
rounded to fp32 before it joins the chain, never contracted into an FMA, so a weight-1 chain is the unweighted chain bit
for bit.  The reductions keep the order and divisors of oracle/full_neighbor.py:
  mean       acc = +0; acc = acc + fl(w_j x_j) in order; acc / fp32(count), count = max(deg, 1) (not the weights' sum)
  mean_self  the same sum, then acc + x[clamp(v)] (the node's own row, weight 1); acc / fp32(count + 1)      (GCN)
  max        m = fl(w_0 x_0); m = fmax(m, fl(w_j x_j)) in order
The pools (max-pool, mean-pool, twomaxpool inference) weight the MLP output z after its ReLU: max_j fl(w_j z_j), or
(Σ_j fl(w_j z_j)) / count.  Implicit entries weigh 1: an empty row's dummy entry and an out-of-range node's dummy entry.
A zero weight makes fl(0 * x) a zero of x's sign; where a max chain meets +0 and -0 as its largest values the sign of
the result is fmaxf's choice and is not part of the contract (every reader of m - the GEMM, the backward's tie test -
treats both zeros alike), so a max is compared with +0 and -0 as one value.

Blocks.  A full-neighbourhood block (oracle/full_neighbor_blocks.py) copies node g's raw row, so entry j of local row u
weighs w[indptr[g] + j], g = src_ids[u].  A sampled block entry e is raw entry indptr[g] + pos_off[e]
(oracle/sampled_blocks_dropout.entry_offsets) and weighs w there.  Blocks therefore reduce the same messages, in the
same order, as the whole graph: their rows are the whole graph's rows bit for bit.

Backward (the effective CSR and its transpose are oracle/full_neighbor_grad.py's).  Each effective entry carries its
forward weight, 1 for the {N} entries (empty rows, the dummy row) and the GCN self entry; a transposed entry carries the
weight of the effective entry it came from: t_weight = w[indptr[i] + slot] for slot >= 0, 1 for slots -1 and -2.
  means  g'[i] = fl(g[i] / count_i); dsrc[j] = +0 + Σ fl(t_weight * g'[i]) over transposed row j, in order (GS_CSR_SUM).
  max    (a) cnt[i][c] = #{entries e of row i : fl(w_e z[e][c]) == m[i][c]}; s[i][c] = dm[i][c] / cnt;
         (b) acc = +0; for each entry of transposed row j, in order, from row i with weight w:
             if fl(w z[j][c]) == m[i][c]: acc = acc + fl(w s[i][c]);  dz[j][c] = acc where z[j][c] > 0, else +0.
         So z_j gets w_j dm / ties at the entries where fl(w_j z_j) == m, and 0 at the others.

Test infrastructure - not imported by the product.
"""
import numpy as np

from . import full_neighbor as fn
from . import full_neighbor_grad as fg
from .aggregate import l2_normalize, relu
from .full_neighbor_blocks import clamp_ids, csr_blocks
from .numerics import gather_clamped
from .sampled_blocks_dropout import entry_offsets

OPS = ("mean", "mean_self", "max")


def _weights(weights, n):
    """weights as float32 [n]; None: all ones."""
    if weights is None:
        return np.ones(n, dtype=np.float32)
    w = np.asarray(weights)
    if w.dtype != np.float32 or w.shape != (n,):
        raise ValueError("weights must be float32 with one value per CSR entry (%d)" % n)
    return w


def csr_aggregate(table, indptr, indices, op, rows=None, weights=None):
    """gs_csr_aggregate_weighted (ops mean, mean_self, max) in the kernel's order, bit for bit.  table: float32 [R, F] or
    uint16 bf16 bits (widened exactly).  Returns float32 [n, F]."""
    if op not in OPS:
        raise ValueError("op must be one of %s" % (OPS,))
    table = np.asarray(table)
    R = table.shape[0]
    indices = np.asarray(indices, dtype=np.int64)
    w = _weights(weights, len(indices))
    nodes, lo, cnt = fn.csr_rows(indptr, indices, R, rows)
    n, F = len(nodes), table.shape[1]
    count = np.maximum(cnt, 1)

    def entry(sel, j):                             # fl(w * x) of entry j of the rows `sel`
        ids = np.full(len(sel), R - 1, dtype=np.int64)
        ws = np.ones(len(sel), dtype=np.float32)
        has = cnt[sel] > 0
        ids[has] = indices[lo[sel][has] + j]
        ws[has] = w[lo[sel][has] + j]
        return (ws[:, None] * gather_clamped(table, ids)).astype(np.float32)

    acc = np.zeros((n, F), dtype=np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        if op == "max":
            acc = entry(np.arange(n), 0)
        for j in range(1 if op == "max" else 0, int(count.max()) if n else 0):
            sel = np.nonzero(count > j)[0]
            x = entry(sel, j)
            acc[sel] = np.fmax(acc[sel], x) if op == "max" else acc[sel] + x
        if op == "max":
            return acc
        if op == "mean_self":
            acc = acc + gather_clamped(table, nodes)
            return acc / (count + 1).astype(np.float32)[:, None]
        return acc / count.astype(np.float32)[:, None]


def dense_reference(table, indptr, indices, op, rows=None, weights=None):
    """The same reduction in float64 from a dense weighted adjacency row: the formula, not the order."""
    table = np.asarray(table, dtype=np.float64)
    R = table.shape[0]
    indices = np.asarray(indices, dtype=np.int64)
    w = _weights(weights, len(indices)).astype(np.float64)
    nodes, lo, cnt = fn.csr_rows(indptr, indices, R, rows)
    out = np.zeros((len(nodes), table.shape[1]))
    for i, (v, a, c) in enumerate(zip(nodes, lo, cnt)):
        ids = indices[a:a + c] if c else np.array([R - 1])
        ws = w[a:a + c] if c else np.ones(1)
        ids = np.where((ids < 0) | (ids >= R), R - 1, ids)
        if op == "max":
            out[i] = (ws[:, None] * table[ids]).max(axis=0)
            continue
        A = np.zeros(R)
        np.add.at(A, ids, ws)                                            # one dense weighted adjacency row
        if op == "mean_self":
            A[v if 0 <= v < R else R - 1] += 1
        out[i] = A @ table / (len(ids) + (op == "mean_self"))
    return out


def effective_weights(indptr, weights, with_self=False):
    """The weights of oracle.full_neighbor_grad.effective_csr's entries: each CSR entry's own, 1 for the {N} entries and
    the with_self entries.  float32."""
    indptr = np.asarray(indptr, dtype=np.int64)
    N = len(indptr) - 1
    w = None if weights is None else np.asarray(weights, dtype=np.float32)
    rows = []
    for i in range(N + 1):
        if i < N and indptr[i + 1] > indptr[i]:
            e = w[indptr[i]:indptr[i + 1]] if w is not None else np.ones(indptr[i + 1] - indptr[i], np.float32)
        else:
            e = np.ones(1, dtype=np.float32)
        rows.append(np.concatenate([e, np.ones(1, np.float32)]) if with_self else e)
    return np.concatenate(rows).astype(np.float32)


def transpose_weights(indptr, indices, weights, with_self=False):
    """The weights of oracle.full_neighbor_grad.csr_transpose's entries, aligned with its t_indices."""
    _, eidx = fg.effective_csr(indptr, indices, with_self)
    return effective_weights(indptr, weights, with_self)[np.argsort(eidx, kind="stable")]


def csr_sum(table, t_indptr, t_indices, t_weights):
    """GS_CSR_SUM over weighted entries, bit for bit: acc = +0; acc = acc + fl(w_j x_j) in order."""
    table = np.asarray(table, dtype=np.float32)
    n = len(t_indptr) - 1
    cnt = np.diff(t_indptr)
    acc = np.zeros((n, table.shape[1]), dtype=np.float32)
    for j in range(int(cnt.max()) if n else 0):
        sel = np.nonzero(cnt > j)[0]
        k = t_indptr[sel] + j
        acc[sel] = acc[sel] + (t_weights[k][:, None] * table[t_indices[k]]).astype(np.float32)
    return acc


def mean_backward(g, indptr, indices, with_self=False, weights=None):
    """d(src) of the weighted mean over the effective rows (mean_self with with_self) for the dense gradient g."""
    t_indptr, t_indices = fg.csr_transpose(indptr, indices, with_self)
    gp = (np.asarray(g, dtype=np.float32) / fg.mean_counts(indptr, with_self)[:, None]).astype(np.float32)
    return csr_sum(gp, t_indptr, t_indices, transpose_weights(indptr, indices, weights, with_self))


def max_backward(z, m, dm, indptr, indices, weights=None):
    """gs_csr_max_backward_weighted, bit for bit: (s, dz), both fp32 [N + 1, F]."""
    z, m, dm = (np.asarray(x, dtype=np.float32) for x in (z, m, dm))
    eptr, eidx = fg.effective_csr(indptr, indices)
    ew = effective_weights(indptr, weights)
    ecnt = np.diff(eptr)
    cnt = np.zeros_like(m)
    for p in range(int(ecnt.max())):
        sel = np.nonzero(ecnt > p)[0]
        k = eptr[sel] + p
        cnt[sel] += (ew[k][:, None] * z[eidx[k]] == m[sel]).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = (dm / cnt).astype(np.float32)
    t_indptr, t_indices = fg.csr_transpose(indptr, indices)
    tw = transpose_weights(indptr, indices, weights)
    tcnt = np.diff(t_indptr)
    acc = np.zeros_like(z)
    for p in range(int(tcnt.max()) if len(tcnt) else 0):
        sel = np.nonzero(tcnt > p)[0]
        k = t_indptr[sel] + p
        i, w = t_indices[k], tw[k][:, None]
        acc[sel] = np.where(w * z[sel] == m[i], acc[sel] + (w * s[i]).astype(np.float32), acc[sel])
    return s, np.where(z > 0, acc, np.float32(0)).astype(np.float32)


def block_weights(indptr, weights, block, offsets=None):
    """The weights of a block's entries, aligned with block["indices"]: weights[indptr[src_ids[u]] + j] for entry j of
    local row u, or + offsets[e] for a sampled block (entry_offsets)."""
    indptr = np.asarray(indptr, dtype=np.int64)
    bptr = np.asarray(block["indptr"], dtype=np.int64)
    cnt = np.diff(bptr)
    u = np.repeat(np.arange(len(cnt)), cnt)
    off = np.arange(len(u)) - bptr[u] if offsets is None else np.asarray(offsets, dtype=np.int64)
    g = np.asarray(block["src_ids"], dtype=np.int64)[u]
    return np.asarray(weights, dtype=np.float32)[indptr[g] + off] if len(u) else np.zeros(0, np.float32)


# ---------------------------------------------------------------- layers and drivers
def _pool_z(agg, h):
    """The pools' MLP output, once per row: relu(h Wm + bm), or twomaxpool's relu(relu(h W1 + b1) W2 + b2)."""
    if agg["type"] == "twomaxpool":
        return relu(relu(h @ agg["W1"] + agg["b1"]).astype(np.float32) @ agg["W2"] + agg["b2"]).astype(np.float32)
    return relu(h @ agg["mlp_weights"] + agg["mlp_bias"]).astype(np.float32)


def _layer_forward(agg, h, graph, rows, concat, last):
    """One layer over graph = (indptr, indices, weights), keeping what the backward reads (as
    oracle.full_neighbor_grad._layer_forward: the pools reduce all N + 1 rows, then read `rows`)."""
    indptr, indices, w = graph
    kind, c = agg["type"], {"h": h}
    if kind == "gcn":
        c["p"] = csr_aggregate(h, indptr, indices, "mean_self", rows, w)
        y = c["p"] @ agg["weights"]
    else:
        if kind == "mean":
            c["p"] = csr_aggregate(h, indptr, indices, "mean", rows, w)
        else:
            c["z"] = _pool_z(agg, h)
            c["p_all"] = csr_aggregate(c["z"], indptr, indices, "mean" if kind == "meanpool" else "max", None, w)
            c["p"] = c["p_all"] if rows is None else c["p_all"][clamp_ids(rows, len(indptr) - 1)]
        c["hs"] = h if rows is None else gather_clamped(h, rows)
        y = fn._combine(c["hs"] @ agg["self_weights"], c["p"] @ agg["neigh_weights"], concat)
    if agg.get("bias") is not None:
        y = y + agg["bias"]
    c["y"] = (y if last else relu(y)).astype(np.float32)
    return c


def _layer_backward(agg, c, dy, graph, rows, concat, last, need_dsrc):
    """(weight gradients {name: array}, d(layer input) [N + 1, in] or None), as oracle.full_neighbor_grad's."""
    indptr, indices, w = graph
    kind = agg["type"]
    n_rows = c["h"].shape[0]
    dz = dy if last else np.where(c["y"] > 0, dy, np.float32(0)).astype(np.float32)
    grads = {}
    if agg.get("bias") is not None:
        grads["bias"] = dz.sum(axis=0)
    dense = (lambda x: x) if rows is None else (lambda x: fg.scatter_rows(x, rows, n_rows))
    if kind == "gcn":
        grads["weights"] = c["p"].T @ dz
        if not need_dsrc:
            return grads, None
        return grads, mean_backward(dense(dz @ agg["weights"].T), indptr, indices, True, w)
    D = agg["self_weights"].shape[1]
    dzs, dzn = (dz[:, :D], dz[:, D:]) if concat else (dz, dz)
    grads["self_weights"] = c["hs"].T @ dzs
    grads["neigh_weights"] = c["p"].T @ dzn
    dp = dense((dzn @ agg["neigh_weights"].T).astype(np.float32))
    if kind == "mean":
        if not need_dsrc:
            return grads, None
        return grads, mean_backward(dp, indptr, indices, False, w) + dense(dzs @ agg["self_weights"].T)
    if kind == "maxpool":
        _, dzp = max_backward(c["z"], c["p_all"], dp, indptr, indices, w)
    else:
        dzp = np.where(c["z"] > 0, mean_backward(dp, indptr, indices, False, w), np.float32(0)).astype(np.float32)
    grads["mlp_weights"] = c["h"].T @ dzp
    grads["mlp_bias"] = dzp.sum(axis=0)
    if not need_dsrc:
        return grads, None
    return grads, dzp @ agg["mlp_weights"].T + dense(dzs @ agg["self_weights"].T)


def layer_graphs(indptr, indices, weights, node_ids, n_layers, mode="whole", fanouts=None, seed=0, call=0):
    """(h0 ids or None, [(graph, rows, src_ids or None)] per layer) of one pass: mode "whole" - every layer over the
    global CSR, the last one's rows node_ids; "blocks" - over csr_blocks' blocks; "sampled" - over the sampled blocks of
    (fanouts, seed, call).  A block layer's graph carries its block weights; the pass reads h0 = the rows ids of the
    table (V_0) instead of the whole table."""
    N = len(indptr) - 1
    w = _weights(weights, len(np.asarray(indices)))
    if mode == "whole":
        ids = np.asarray(node_ids, dtype=np.int64).reshape(-1)
        return None, [((indptr, indices, w), ids if l == n_layers - 1 else None, None) for l in range(n_layers)]
    if mode == "blocks":
        blocks, offs = csr_blocks(indptr, indices, clamp_ids(node_ids, N), n_layers), [None] * n_layers
    else:
        blocks, offs = entry_offsets(indptr, indices, node_ids, fanouts, seed, call)
    out = [((b["indptr"], b["indices"], block_weights(indptr, w, b, o)), b["rows"], b["src_ids"])
           for b, o in zip(blocks, offs)]
    return blocks[0]["src_ids"], out


def embeddings(features, indptr, indices, weights, aggregators, concat, node_ids=None, normalize=True, mode="whole",
               fanouts=None, seed=0, call=0):
    """The weighted layer loop: float32 [len(node_ids), w] (node_ids None: all N nodes, mode "whole" only)."""
    h = np.asarray(features, dtype=np.float32)
    N = h.shape[0] - 1
    node_ids = np.arange(N) if node_ids is None else node_ids
    v0, graphs = layer_graphs(indptr, indices, weights, node_ids, len(aggregators), mode, fanouts, seed, call)
    if v0 is not None:
        h = gather_clamped(h, v0)
    L = len(aggregators)
    for l, (agg, (graph, rows, _)) in enumerate(zip(aggregators, graphs)):
        h = _layer_forward(agg, h, graph, rows, concat, l == L - 1)["y"]
    return l2_normalize(h) if normalize else h


def loss_grads(features, indptr, indices, weights, aggregators, concat, node_ids, labels, pred_weights, pred_bias,
               sigmoid_loss=False, weight_decay=0.0, identity_dim=0, mode="whole", fanouts=None, seed=0, call=0):
    """The supervised step over weighted edges, as oracle.full_neighbor_grad.full_neighbor_loss_grads (same returns)."""
    h = np.asarray(features, dtype=np.float32)
    labels = np.asarray(labels, dtype=np.float64)
    L = len(aggregators)
    v0, graphs = layer_graphs(indptr, indices, weights, node_ids, L, mode, fanouts, seed, call)
    if v0 is not None:
        h = gather_clamped(h, v0)
    caches = []
    for l, (agg, (graph, rows, _)) in enumerate(zip(aggregators, graphs)):
        caches.append(_layer_forward(agg, h, graph, rows, concat, l == L - 1))
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
        g, dsrc = _layer_backward(agg, caches[l], dy, graph, rows, concat, l == L - 1, l > 0 or identity_dim > 0)
        for k in g:
            if weight_decay and k not in ("mlp_weights", "mlp_bias"):
                g[k] = g[k] + weight_decay * agg[k]
                loss += 0.5 * weight_decay * float((np.asarray(agg[k], np.float64) ** 2).sum())
        grads[l] = g
        if l > 0:
            dy = dsrc.astype(np.float32)
        elif identity_dim > 0:
            d = dsrc[:, :identity_dim]
            demb = d if src_ids is None else fg.scatter_rows(d, src_ids, np.asarray(features).shape[0])
    return float(loss), grads, head, demb
