"""Full-neighbourhood training with dropout: the contract of gs_csr_aggregate_dropout, gs_csr_transpose's t_slot, the
positioned gs_dropout_apply and the `dropout=p` argument of the full_neighbor_* training methods.  Plain numpy, fp32,
in kernel order.  The unmasked layer loop is oracle/full_neighbor.py's; every rule here only adds masks to it.

Sites.  One call with rate p > 0 numbers its sites from the model's dropout_counter (full_neighbor_site_plan): per
layer "neigh" then "self" (mean, gcn) or "mlp" (max-pool, mean-pool), then "head" (supervised only).  Each site is the
(seed, call, p) Philox rule of oracle/dropout.py; the counter advances by the number of sites.  What is new is the
positions, all of them GLOBAL identities, so a minibatch block masks every element as the whole-graph pass does:
  neigh  entry j of node v's raw CSR row (out-of-range entries included; they read the dummy row): indptr[v] + j;
         the implicit dummy entry of an empty row, of a node outside [0, N) or of the dummy node N: nnz + v (v = N for
         the last two), nnz = len(indices) of the global CSR;
  self   the mean's self-branch row of node v, and the GCN's own row inside mean_self: v;
  mlp    the pools' MLP input row of node v: v (the full path runs the MLP once per node, so its input mask is per node;
         a per-edge mask would mean one MLP per edge, the cost this path exists to avoid);
  head   row r of node_ids: r, as on the sampled path.
Per-edge neighbour masks follow the reference, where every sampled neighbour copy is dropped independently: a hub's row
is not removed from all its readers at once.

Position map.  A kernel over a local CSR names local row r's global node g(r) = pos_ids[r] (pos_ids None: r), r first
clamped to the dummy row n_nodes, and entry j of it pos_indptr[g] + j; the whole graph passes (indptr, None, nnz), a
block (global indptr, block src_ids, global nnz).  Blocks keep raw rows in CSR order, so block entry j is global entry j.

Arithmetic (oracle/dropout.py): a kept element is x / keep (keep = fp32(1 - p)), a dropped one 0; the reductions' sum
order and divisors are gs_csr_aggregate's with each masked element in place of the raw one (bf16 sources widened first).

Backward: every mask is regenerated, none stored.
  t_slot   gs_csr_transpose's slot of each transposed entry within its forward row i: j, -1 for the implicit dummy entry,
           -2 for a with_self entry;
  mean/gcn dsrc[j] = +0 + sum over transposed row j, in order, of drop(site, pos, g[i] / count_i) - the entry's own
           neigh position, or the self site at g(i) for a -2 entry (GS_CSR_SUM with the flag);
  self     the mean's self-branch gradient, and the pools' dX = dZ Wm^T, masked by the node mask of their dense row;
  dWm      X^T dZ with X the masked MLP input.

Test infrastructure - not imported by the product.
"""
import numpy as np

from .aggregate import l2_normalize, relu
from .dropout import apply as drop_rows
from .dropout import keep_mask, keep_prob
from .full_neighbor import _combine, csr_aggregate, csr_rows
from .full_neighbor_blocks import clamp_ids, csr_blocks
from .full_neighbor_grad import effective_csr, max_backward, mean_counts, scatter_rows
from .numerics import gather_clamped


def site_plan(kind, n_layers, head=False):
    """[(layer, role)]: per layer ("neigh", "self") for mean / gcn or ("mlp",) for the pools, then (None, "head")."""
    roles = ("mlp",) if kind in ("maxpool", "meanpool") else ("neigh", "self")
    return [(l, r) for l in range(n_layers) for r in roles] + ([(None, "head")] if head else [])


def sites(kind, n_layers, head, seed, call0, rate):
    """{(layer, role): (seed, call, rate)} with calls numbered from call0 in site_plan order."""
    return {k: (seed, call0 + i, rate) for i, k in enumerate(site_plan(kind, n_layers, head))}


def _drop(x, site, pos):
    """where(mask(site, pos), x / keep, 0) for x [len(pos), F] in fp32."""
    seed, call, rate = site
    m = keep_mask(seed, call, rate, pos, x.shape[1])
    return np.where(m, np.asarray(x, np.float32) / keep_prob(rate), np.float32(0)).astype(np.float32)


def global_nodes(local, n_nodes, pos_ids):
    """g(r): local rows clamped to the dummy row n_nodes, then through pos_ids."""
    local = np.asarray(local, dtype=np.int64)
    vc = np.where((local < 0) | (local >= n_nodes), n_nodes, local)
    return vc if pos_ids is None else np.asarray(pos_ids, np.int64)[vc]


def row_bases(indptr, indices, rows, pos_map, R):
    """(nodes, lo, cnt, g, base): the rows of csr_rows, their global nodes and the position of their entry 0."""
    pos_indptr, pos_ids, pos_nnz = pos_map
    nodes, lo, cnt = csr_rows(indptr, indices, R, rows)
    g = global_nodes(nodes, len(indptr) - 1, pos_ids)
    pos_indptr = np.asarray(pos_indptr, np.int64)
    base = np.where(cnt > 0, pos_indptr[np.minimum(g, len(pos_indptr) - 1)], pos_nnz + g)
    return nodes, lo, cnt, g, base


def csr_aggregate_dropout(table, indptr, indices, op, neigh, self_site, pos_map, rows=None):
    """gs_csr_aggregate_dropout (ops "mean", "mean_self") bit for bit: fp32 [n, F]."""
    table = np.asarray(table)
    R, F = table.shape
    indices = np.asarray(indices, dtype=np.int64)
    nodes, lo, cnt, g, base = row_bases(indptr, indices, rows, pos_map, R)
    count = np.maximum(cnt, 1)
    acc = np.zeros((len(nodes), F), dtype=np.float32)
    for j in range(int(count.max()) if len(nodes) else 0):
        sel = np.nonzero(count > j)[0]
        ids = np.full(len(sel), R - 1, dtype=np.int64)
        has = cnt[sel] > 0
        ids[has] = indices[lo[sel][has] + j]
        acc[sel] = acc[sel] + _drop(gather_clamped(table, ids), neigh, base[sel] + j)
    if op == "mean_self":
        acc = acc + _drop(gather_clamped(table, nodes), self_site, g)
        return acc / (count + 1).astype(np.float32)[:, None]
    if op != "mean":
        raise ValueError(op)
    return acc / count.astype(np.float32)[:, None]


def csr_transpose_slots(indptr, indices, with_self=False):
    """gs_csr_transpose with t_slot: (t_indptr, t_indices, t_slot), the last two int64 [effective entries]."""
    indptr = np.asarray(indptr, dtype=np.int64)
    eptr, eidx = effective_csr(indptr, indices, with_self)
    N = len(eptr) - 2
    src = np.repeat(np.arange(N + 1), np.diff(eptr))
    slot = np.concatenate([np.arange(n) for n in np.diff(eptr)]).astype(np.int64) if len(eidx) else eidx
    cnt = np.concatenate([np.diff(indptr), [0]])[src]
    slot = np.where(with_self & (slot == np.diff(eptr)[src] - 1), -2, np.where(cnt > 0, slot, -1))
    order = np.argsort(eidx, kind="stable")
    t_indptr = np.zeros(N + 2, dtype=np.int64)
    t_indptr[1:] = np.cumsum(np.bincount(eidx, minlength=N + 1))
    return t_indptr, src[order].astype(np.int64), slot[order].astype(np.int64)


def csr_sum_dropout(table, t_indptr, t_indices, t_slot, neigh, self_site, pos_map):
    """GS_CSR_SUM of gs_csr_aggregate_dropout bit for bit: acc = +0; acc += drop(entry site, pos, x_i) in order."""
    pos_indptr, pos_ids, pos_nnz = pos_map
    table = np.asarray(table, dtype=np.float32)
    n, F = len(t_indptr) - 1, table.shape[1]
    cnt = np.diff(t_indptr)
    acc = np.zeros((n, F), dtype=np.float32)
    for j in range(int(cnt.max()) if n else 0):
        sel = np.nonzero(cnt > j)[0]
        i = np.asarray(t_indices, np.int64)[t_indptr[sel] + j]
        s = np.asarray(t_slot, np.int64)[t_indptr[sel] + j]
        g = global_nodes(i, table.shape[0] - 1, pos_ids)
        pos = np.where(s >= 0, np.asarray(pos_indptr, np.int64)[g] + s, np.where(s == -1, pos_nnz + g, g))
        x = table[i]
        acc[sel] = acc[sel] + np.where((s == -2)[:, None], _drop(x, self_site, pos), _drop(x, neigh, pos))
    return acc


def mean_backward_dropout(g, indptr, indices, with_self, neigh, self_site, pos_map):
    """d(src) of the masked mean over the effective rows for the dense gradient g [N + 1, w]."""
    t_indptr, t_indices, t_slot = csr_transpose_slots(indptr, indices, with_self)
    gp = (np.asarray(g, dtype=np.float32) / mean_counts(indptr, with_self)[:, None]).astype(np.float32)
    return csr_sum_dropout(gp, t_indptr, t_indices, t_slot, neigh, self_site, pos_map)


def _layer_forward(agg, h, indptr, indices, rows, concat, last, s, pos_map, table_csr=None):
    """One masked layer, keeping what the backward reads.  s: {"neigh", "self"} or {"mlp"} sites.  table_csr: (indptr,
    indices, rows, pos_map) the means read h through instead (a block's layer 0); the rest runs in the graph's space."""
    kind, c = agg["type"], {"h": h}
    n_nodes = len(indptr) - 1
    t_ptr, t_idx, t_rows, t_map = table_csr if table_csr is not None else (indptr, indices, rows, pos_map)
    if kind == "gcn":
        c["p"] = csr_aggregate_dropout(h, t_ptr, t_idx, "mean_self", s["neigh"], s["self"], t_map, t_rows)
        y = c["p"] @ agg["weights"]
    else:
        if kind == "mean":
            hs = h if t_rows is None else gather_clamped(h, t_rows)
            sel = np.arange(h.shape[0]) if t_rows is None else t_rows
            c["hs"] = _drop(hs, s["self"], global_nodes(sel, len(t_ptr) - 1, t_map[1]))
            c["p"] = csr_aggregate_dropout(h, t_ptr, t_idx, "mean", s["neigh"], s["self"], t_map, t_rows)
        else:
            c["hs"] = h if rows is None else gather_clamped(h, rows)
            c["x"] = _drop(h, s["mlp"], global_nodes(np.arange(h.shape[0]), n_nodes, pos_map[1]))
            c["z"] = relu(c["x"] @ agg["mlp_weights"] + agg["mlp_bias"]).astype(np.float32)
            c["p_all"] = csr_aggregate(c["z"], indptr, indices, "max" if kind == "maxpool" else "mean")
            c["p"] = c["p_all"] if rows is None else c["p_all"][rows]
        y = _combine(c["hs"] @ agg["self_weights"], c["p"] @ agg["neigh_weights"], concat)
    if agg.get("bias") is not None:
        y = y + agg["bias"]
    c["y"] = (y if last else relu(y)).astype(np.float32)
    return c


def _layer_backward(agg, c, dy, indptr, indices, rows, concat, last, need_dsrc, s, pos_map):
    """(weight gradients, d(layer input) [N + 1, in] or None), every mask regenerated."""
    kind = agg["type"]
    n_rows = c["h"].shape[0]
    dz = dy if last else np.where(c["y"] > 0, dy, np.float32(0)).astype(np.float32)
    grads = {}
    dense = (lambda x: x) if rows is None else (lambda x: scatter_rows(x, rows, n_rows))
    node_mask = global_nodes(np.arange(n_rows), len(indptr) - 1, pos_map[1])
    if kind == "gcn":
        grads["weights"] = c["p"].T @ dz
        if not need_dsrc:
            return grads, None
        return grads, mean_backward_dropout(dense(dz @ agg["weights"].T), indptr, indices, True, s["neigh"], s["self"],
                                            pos_map)
    D = agg["self_weights"].shape[1]
    dzs, dzn = (dz[:, :D], dz[:, D:]) if concat else (dz, dz)
    grads["self_weights"] = c["hs"].T @ dzs
    grads["neigh_weights"] = c["p"].T @ dzn
    dp = dense((dzn @ agg["neigh_weights"].T).astype(np.float32))
    if kind == "mean":
        if not need_dsrc:
            return grads, None
        dself = _drop(dense(dzs @ agg["self_weights"].T), s["self"], node_mask)
        return grads, mean_backward_dropout(dp, indptr, indices, False, s["neigh"], s["self"], pos_map) + dself
    if kind == "maxpool":
        _, dzp = max_backward(c["z"], c["p_all"], dp, indptr, indices)
    else:
        from .full_neighbor_grad import mean_backward
        dzp = np.where(c["z"] > 0, mean_backward(dp, indptr, indices), np.float32(0)).astype(np.float32)
    grads["mlp_weights"] = c["x"].T @ dzp
    grads["mlp_bias"] = dzp.sum(axis=0)
    if not need_dsrc:
        return grads, None
    return grads, _drop(dzp @ agg["mlp_weights"].T, s["mlp"], node_mask) + dense(dzs @ agg["self_weights"].T)


def _layer_sites(all_sites, l):
    return {role: v for (layer, role), v in all_sites.items() if layer == l}


def full_neighbor_outputs(features, indptr, indices, aggregators, concat, node_ids, all_sites, normalize=True):
    """The whole-graph training forward with masks (no head): fp32 [len(node_ids), w].  all_sites: sites(...)."""
    h = np.asarray(features, dtype=np.float32)
    nnz = len(indices)
    node_ids = clamp_ids(node_ids, len(indptr) - 1)
    L = len(aggregators)
    for l, agg in enumerate(aggregators):
        last = l == L - 1
        h = _layer_forward(agg, h, indptr, indices, node_ids if last else None, concat, last, _layer_sites(all_sites, l),
                           (indptr, None, nnz))["y"]
    return l2_normalize(h) if normalize else h


def block_outputs(features, indptr, indices, aggregators, concat, seeds, all_sites, normalize=True):
    """full_neighbor_outputs over csr_blocks: each block masks through (global indptr, src_ids, global nnz); layer 0's
    means read the global table through the global CSR with rows = V_1 (pos_ids None), the pools' MLP V_0's rows."""
    features = np.asarray(features, dtype=np.float32)
    nnz, N = len(indices), len(indptr) - 1
    L = len(aggregators)
    blocks = csr_blocks(indptr, indices, seeds, L)
    h = None
    for l, agg in enumerate(aggregators):
        b, last, s = blocks[l], l == L - 1, _layer_sites(all_sites, l)
        bmap = (indptr, b["src_ids"], nnz)
        if l == 0 and agg["type"] in ("mean", "gcn"):
            v1 = blocks[1]["src_ids"] if L > 1 else clamp_ids(seeds, N)
            h = _layer_forward(agg, features, b["indptr"], b["indices"], b["rows"], concat, last, s, bmap,
                               table_csr=(indptr, indices, v1, (indptr, None, nnz)))["y"]
        else:
            src = gather_clamped(features, b["src_ids"]) if l == 0 else h
            h = _layer_forward(agg, src, b["indptr"], b["indices"], b["rows"], concat, last, s, bmap)["y"]
    return l2_normalize(h) if normalize else h


def full_neighbor_loss_grads(features, indptr, indices, aggregators, concat, node_ids, labels, pred_weights, pred_bias,
                             all_sites, sigmoid_loss=False, weight_decay=0.0, identity_dim=0):
    """oracle.full_neighbor_grad.full_neighbor_loss_grads with the masks of all_sites (sites(kind, L, True, ...)): the
    same returns."""
    h = np.asarray(features, dtype=np.float32)
    nnz = len(indices)
    pmap = (indptr, None, nnz)
    node_ids = clamp_ids(node_ids, len(indptr) - 1)
    labels = np.asarray(labels, dtype=np.float64)
    L = len(aggregators)
    caches = []
    for l, agg in enumerate(aggregators):
        last = l == L - 1
        c = _layer_forward(agg, h, indptr, indices, node_ids if last else None, concat, last, _layer_sites(all_sites, l),
                           pmap)
        caches.append(c)
        h = c["y"]
    head_site = all_sites[(None, "head")]
    out32 = drop_rows(l2_normalize(h), *head_site)
    out = out32.astype(np.float64)
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
        agg, last = aggregators[l], l == L - 1
        g, dsrc = _layer_backward(agg, caches[l], dy, indptr, indices, node_ids if last else None, concat, last,
                                  l > 0 or identity_dim > 0, _layer_sites(all_sites, l), pmap)
        for k in g:
            if weight_decay and k not in ("mlp_weights", "mlp_bias"):
                g[k] = g[k] + weight_decay * agg[k]
                loss += 0.5 * weight_decay * float((np.asarray(agg[k], np.float64) ** 2).sum())
        grads[l] = g
        if l > 0:
            dy = dsrc.astype(np.float32)
        elif identity_dim > 0:
            demb = dsrc[:, :identity_dim]
    return float(loss), grads, head, demb


def dense_masked_mean(table, indptr, indices, op, neigh, self_site, rows=None):
    """The whole-graph masked mean in float64 from an explicit per-edge mask tensor M [n, max entries, F] (the formula,
    not the order): out[i] = sum_j M[i, j] * x[src(i, j)] / keep / count_i (+ the masked self row for mean_self)."""
    table = np.asarray(table, dtype=np.float64)
    R, F = table.shape
    indptr = np.asarray(indptr, np.int64)
    indices = np.asarray(indices, np.int64)
    N, nnz = len(indptr) - 1, len(indices)
    nodes = np.arange(N + 1) if rows is None else np.asarray(rows, np.int64)
    out = np.zeros((len(nodes), F))
    for i, v in enumerate(nodes):
        inside = 0 <= v < N
        c = max(indptr[v + 1] - indptr[v], 0) if inside else 0
        if c:
            src, pos = indices[indptr[v]:indptr[v] + c], indptr[v] + np.arange(c)
        else:
            src, pos = np.array([R - 1]), np.array([nnz + (v if inside else N)])
        src = np.where((src < 0) | (src >= R), R - 1, src)
        M = keep_mask(*neigh, pos, F)
        acc = (M * table[src]).sum(axis=0) / np.float64(keep_prob(neigh[2]))
        if op == "mean_self":
            vv = v if inside else N
            acc += keep_mask(*self_site, [vv], F)[0] * table[min(vv, R - 1)] / np.float64(keep_prob(self_site[2]))
            c = max(c, 1) + 1
        out[i] = acc / max(c, 1)
    return out
