"""Full-batch training over whole neighbourhoods: the backward contract of gs_csr_transpose, the GS_CSR_SUM op of
gs_csr_aggregate, gs_csr_max_backward and SupervisedGraphsage.full_neighbor_train_step.  Plain numpy, fp32, in kernel
order.  The forward is oracle/full_neighbor.py's layer loop, unchanged.

The effective CSR (N + 1 rows; the forward reads exactly these source rows, in this order):
  row i < N: indices[indptr[i] .. indptr[i+1]) in CSR order, an entry outside [0, N] replaced by N (the forward's clamp);
             an empty row (indptr[i+1] <= indptr[i]) is {N};
  row N (the dummy node): {N};
  with_self (GCN, the mean_self rule): every row i then has its own id i appended.
The transpose: row j holds the rows i of every effective entry equal to j, in ascending i, the entries of one row in their
CSR order - a stable sort of the (destination, source row) pairs by destination.

Backward of the means (mean, GCN, mean-pool):  g'[i] = fl(g[i] / count_i), count_i the forward's divisor (max(cnt, 1),
  + 1 for GCN);  dsrc[j] = +0 + sum of g'[i] over transposed row j, in order (GS_CSR_SUM).  A node that is nobody's
  neighbour gets exactly 0.
Backward of the max (TensorFlow's reduce_max gradient, as pool_branch_backward applies it on sampled rows):
  (a) cnt[i][c] = #{entries e of effective row i : z[e][c] == m[i][c]} (duplicates counted); s[i][c] = dm[i][c] / cnt;
  (b) acc = +0; for i in transposed row j, in order: if z[j][c] == m[i][c]: acc += s[i][c];
      dz[j][c] = acc where z[j][c] > 0, else +0 (the ReLU of the Dense layer that made z).
The last layer reads only the rows of node_ids (duplicates allowed): their gradients are scattered into a dense
[N+1, w] gradient (ops.embedding_grad, group 1; its fixed summation order is oracle/sparse_grad.py's
embedding_grad_reference, bit for bit - this module sums in fp64, so compare with it within a tolerance) before the
above runs.  With identity_dim = d > 0 the layer-0 table's columns [0, d) are trained: their gradient is column [0, d) of
the layer-0 source gradient.  Feature columns are not trainable.

Test infrastructure - not imported by the product.
"""
import numpy as np

from .aggregate import l2_normalize, relu
from .full_neighbor import _combine, csr_aggregate
from .numerics import gather_clamped


def effective_csr(indptr, indices, with_self=False):
    """(eptr int64 [N + 2], eidx int64): the effective CSR above."""
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int64)
    N = len(indptr) - 1
    rows = []
    for i in range(N + 1):
        if i < N and indptr[i + 1] > indptr[i]:
            e = indices[indptr[i]:indptr[i + 1]]
            e = np.where((e < 0) | (e > N), N, e)
        else:
            e = np.array([N], dtype=np.int64)
        rows.append(np.concatenate([e, [i]]) if with_self else e)
    eptr = np.zeros(N + 2, dtype=np.int64)
    eptr[1:] = np.cumsum([len(r) for r in rows])
    return eptr, np.concatenate(rows).astype(np.int64)


def csr_transpose(indptr, indices, with_self=False):
    """gs_csr_transpose: (t_indptr int64 [N + 2], t_indices int64 [effective entries])."""
    eptr, eidx = effective_csr(indptr, indices, with_self)
    N = len(eptr) - 2
    src = np.repeat(np.arange(N + 1), np.diff(eptr))
    order = np.argsort(eidx, kind="stable")
    t_indptr = np.zeros(N + 2, dtype=np.int64)
    t_indptr[1:] = np.cumsum(np.bincount(eidx, minlength=N + 1))
    return t_indptr, src[order].astype(np.int64)


def csr_sum(table, t_indptr, t_indices):
    """GS_CSR_SUM over every row of (t_indptr, t_indices), bit for bit: acc = +0; acc += x_j in order."""
    table = np.asarray(table, dtype=np.float32)
    n = len(t_indptr) - 1
    cnt = np.diff(t_indptr)
    acc = np.zeros((n, table.shape[1]), dtype=np.float32)
    for j in range(int(cnt.max()) if n else 0):
        sel = np.nonzero(cnt > j)[0]
        acc[sel] = acc[sel] + table[t_indices[t_indptr[sel] + j]]
    return acc


def mean_counts(indptr, with_self=False):
    """count_i of the forward's division for the N + 1 effective rows, as fp32."""
    indptr = np.asarray(indptr, dtype=np.int64)
    cnt = np.maximum(np.diff(indptr), 1)
    return (np.concatenate([cnt, [1]]) + (1 if with_self else 0)).astype(np.float32)


def mean_backward(g, indptr, indices, with_self=False):
    """d(src) of m = mean over the effective rows (mean_self with with_self) for the dense gradient g [N + 1, w]."""
    t_indptr, t_indices = csr_transpose(indptr, indices, with_self)
    gp = (np.asarray(g, dtype=np.float32) / mean_counts(indptr, with_self)[:, None]).astype(np.float32)
    return csr_sum(gp, t_indptr, t_indices)


def max_backward(z, m, dm, indptr, indices):
    """gs_csr_max_backward, bit for bit: (s, dz), both fp32 [N + 1, F]."""
    z, m, dm = (np.asarray(x, dtype=np.float32) for x in (z, m, dm))
    eptr, eidx = effective_csr(indptr, indices)
    n = len(eptr) - 1
    cnt = np.zeros_like(m)
    for i in range(n):
        cnt[i] = (z[eidx[eptr[i]:eptr[i + 1]]] == m[i]).sum(axis=0)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = (dm / cnt).astype(np.float32)
    t_indptr, t_indices = csr_transpose(indptr, indices)
    dz = np.zeros_like(z)
    for j in range(n):
        acc = np.zeros(z.shape[1], dtype=np.float32)
        for i in t_indices[t_indptr[j]:t_indptr[j + 1]]:
            acc = np.where(z[j] == m[i], acc + s[i], acc).astype(np.float32)
        dz[j] = np.where(z[j] > 0, acc, np.float32(0))
    return s, dz


def scatter_rows(x, rows, n_rows):
    """The dense [n_rows, w] gradient of gather_clamped(h, rows): duplicate rows summed (ops.embedding_grad, group 1)."""
    out = np.zeros((n_rows, x.shape[1]), dtype=np.float64)
    np.add.at(out, np.asarray(rows, dtype=np.int64), np.asarray(x, dtype=np.float64))
    return out.astype(np.float32)


def _layer_forward(agg, h, indptr, indices, rows, concat, last):
    """oracle.full_neighbor.layer, keeping what the backward reads.  Pools compute their max / mean for all N + 1 rows
    (the backward needs every row's max) and read the rows of `rows` from it - the same values."""
    kind, c = agg["type"], {"h": h}
    hs = h if rows is None else gather_clamped(h, rows)
    if kind == "gcn":
        c["p"] = csr_aggregate(h, indptr, indices, "mean_self", rows)
        y = c["p"] @ agg["weights"]
    else:
        if kind == "mean":
            c["p"] = csr_aggregate(h, indptr, indices, "mean", rows)
        else:
            c["z"] = relu(h @ agg["mlp_weights"] + agg["mlp_bias"]).astype(np.float32)
            c["p_all"] = csr_aggregate(c["z"], indptr, indices, "max" if kind == "maxpool" else "mean")
            c["p"] = c["p_all"] if rows is None else c["p_all"][rows]
        c["hs"] = hs
        y = _combine(hs @ agg["self_weights"], c["p"] @ agg["neigh_weights"], concat)
    if agg.get("bias") is not None:
        y = y + agg["bias"]
    c["y"] = (y if last else relu(y)).astype(np.float32)
    return c


def _layer_backward(agg, c, dy, indptr, indices, rows, concat, last, need_dsrc):
    """(weight gradients {name: array}, d(layer input) [N + 1, in] or None)."""
    kind = agg["type"]
    n_rows = c["h"].shape[0]
    dz = dy if last else np.where(c["y"] > 0, dy, np.float32(0)).astype(np.float32)
    grads = {}
    if agg.get("bias") is not None:
        grads["bias"] = dz.sum(axis=0)
    dense = (lambda x: x) if rows is None else (lambda x: scatter_rows(x, rows, n_rows))
    if kind == "gcn":
        grads["weights"] = c["p"].T @ dz
        if not need_dsrc:
            return grads, None
        return grads, mean_backward(dense(dz @ agg["weights"].T), indptr, indices, with_self=True)
    D = agg["self_weights"].shape[1]
    dzs, dzn = (dz[:, :D], dz[:, D:]) if concat else (dz, dz)
    grads["self_weights"] = c["hs"].T @ dzs
    grads["neigh_weights"] = c["p"].T @ dzn
    dp = dense((dzn @ agg["neigh_weights"].T).astype(np.float32))
    if kind == "mean":
        if not need_dsrc:
            return grads, None
        return grads, mean_backward(dp, indptr, indices) + dense(dzs @ agg["self_weights"].T)
    if kind == "maxpool":
        _, dzp = max_backward(c["z"], c["p_all"], dp, indptr, indices)
    else:
        dzp = np.where(c["z"] > 0, mean_backward(dp, indptr, indices), np.float32(0)).astype(np.float32)
    grads["mlp_weights"] = c["h"].T @ dzp
    grads["mlp_bias"] = dzp.sum(axis=0)
    if not need_dsrc:
        return grads, None
    return grads, dzp @ agg["mlp_weights"].T + dense(dzs @ agg["self_weights"].T)


def full_neighbor_loss_grads(features, indptr, indices, aggregators, concat, node_ids, labels, pred_weights, pred_bias,
                             sigmoid_loss=False, weight_decay=0.0, identity_dim=0):
    """The supervised full-batch step: loss and gradients of SupervisedGraphsage.full_neighbor_loss.  features: the
    model's [N+1, d + F] layer-0 table (embeddings first when identity_dim = d > 0).  aggregators: oracle dicts as
    oracle.full_neighbor.layer takes them.  Returns (loss, [per-layer grad dicts], {"weights", "bias"} of the head,
    d(embeddings) [N+1, d] or None).  Weight decay covers every aggregator's own variables and the head (not the pools'
    MLP), as the sampled step."""
    h = np.asarray(features, dtype=np.float32)
    node_ids = np.asarray(node_ids, dtype=np.int64).reshape(-1)
    labels = np.asarray(labels, dtype=np.float64)
    L = len(aggregators)
    caches = []
    for l, agg in enumerate(aggregators):
        last = l == L - 1
        c = _layer_forward(agg, h, indptr, indices, node_ids if last else None, concat, last)
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
    head = {"weights": out.T @ dlog, "bias": dlog.sum(axis=0)}
    decayed = [pred_weights, pred_bias]
    grads = [dict() for _ in aggregators]
    if weight_decay:
        head["weights"] = head["weights"] + weight_decay * pred_weights
        head["bias"] = head["bias"] + weight_decay * pred_bias
    loss += 0.5 * weight_decay * sum(float((np.asarray(v, np.float64) ** 2).sum()) for v in decayed)
    dout = dlog @ np.asarray(pred_weights, np.float64).T
    y64 = h.astype(np.float64)
    nrm = np.sqrt(np.maximum((y64 * y64).sum(axis=1, keepdims=True), 1e-12))
    dy = (dout / nrm - y64 * ((dout * y64).sum(axis=1, keepdims=True)) / nrm ** 3).astype(np.float32)
    demb = None
    for l in range(L - 1, -1, -1):
        agg, last = aggregators[l], l == L - 1
        need = l > 0 or identity_dim > 0
        g, dsrc = _layer_backward(agg, caches[l], dy, indptr, indices, node_ids if last else None, concat, last, need)
        grads[l] = g
        if weight_decay:
            for k in g:
                if k not in ("mlp_weights", "mlp_bias"):
                    g[k] = g[k] + weight_decay * agg[k]
                    loss += 0.5 * weight_decay * float((np.asarray(agg[k], np.float64) ** 2).sum())
        if l > 0:
            dy = dsrc.astype(np.float32)
        elif identity_dim > 0:
            demb = dsrc[:, :identity_dim]
    return float(loss), grads, head, demb
