"""Minibatches over whole neighbourhoods: the contract of gs_csr_blocks (ops.csr_blocks) and of the
full_neighbor_minibatch_* methods.  Plain numpy, in the kernels' order.

For a CSR over nodes 0..N-1 (the dummy node is N) and L layers, csr_blocks builds the receptive field of the seeds:
  seeds are clamped: an id outside [0, N) becomes N (as full_neighbor_outputs does);
  V_L = the seeds, in the order given, duplicates kept;
  V_l (l = L-1 .. 0) = sorted-unique(V_{l+1}  u  every entry of the RAW CSR rows of V_{l+1}'s nodes, an entry outside
        [0, N) mapped to N  u  {N}).  Ascending order puts N last: the [n+1, .] table layout the kernels expect.
Block l (input space V_l, output space V_{l+1}):
  src_ids  int32 V_l;
  indptr   int64, |V_l| entries: one CSR row per local node but the last (the dummy is implicit as the last local row, as
           in the global CSR).  A local node in V_{l+1} gets its raw row, entries relabelled to their position in V_l, in
           CSR order; every other row is empty.  A row empty in the global CSR stays empty, so the kernel reads the local
           last row - N's image - and the {N} rule holds;
  indices  int32 local ids;
  rows     int32 positions in V_l of the layer's output nodes: V_{l+1}'s (ascending, the dummy last) for l < L-1, the
           clamped seeds' (in seed order, duplicates kept) for l = L-1.

Why the blocks give the SAME BITS as the whole-graph pass (oracle/full_neighbor.py with node_ids = seeds): every
output element of a layer is one chain over a fixed list of source rows - the reduction's entries in CSR order, then a
GEMM row over the row's own K inputs.  The chain of output node v at layer l reads only v's CSR row and v itself; both
are in V_l by construction (V_{l+1} is a subset of V_l, and so is every entry of V_{l+1}'s rows), relabelling is
monotone, and an empty row or a clamped entry reads the dummy, which is V_l's last row.  So for every node of V_{l+1}
the block computes the same chain over the same values as the whole-graph layer; by induction from the features
(layer 0 reads the global table), every layer's rows equal the whole graph's rows of V_{l+1}.  The GCN self entry is
read by local id: v's position in V_l, present because V_{l+1} is a subset of V_l.  Rows outside V_{l+1} are not
computed; nothing downstream of the seeds reads them.

The backward runs each block's own transpose (oracle/full_neighbor_grad.py on the local CSR): a node outside V_{l+1} has
an empty local row, so it reads only the dummy and receives a zero gradient, as its row does in the whole-graph pass.
Layer 0's source gradient (identity_dim > 0) is formed in V_0's local space and scattered to the table through src_ids.

Test infrastructure - not imported by the product.
"""
import numpy as np

from .aggregate import l2_normalize, relu
from .full_neighbor import layer
from .full_neighbor_grad import _layer_backward, _layer_forward, scatter_rows
from .numerics import gather_clamped


def clamp_ids(ids, n_nodes):
    ids = np.asarray(ids, dtype=np.int64).reshape(-1)
    return np.where((ids < 0) | (ids >= n_nodes), n_nodes, ids)


def csr_blocks(indptr, indices, seeds, n_layers):
    """The L blocks above: a list, index l = layer l, of dicts {src_ids, indptr, indices, rows}."""
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int64)
    N = len(indptr) - 1

    def raw_row(v):
        lo, hi = indptr[v], indptr[v + 1]
        return clamp_ids(indices[lo:max(lo, hi)], N)

    blocks = [None] * n_layers
    nxt = clamp_ids(seeds, N)
    for l in range(n_layers - 1, -1, -1):
        members = np.unique(nxt)
        rows_of = {int(v): raw_row(v) for v in members if v < N}
        V = np.unique(np.concatenate([members, np.array([N], np.int64)] + list(rows_of.values())))
        pos = np.full(N + 1, -1, dtype=np.int64)
        pos[V] = np.arange(len(V))
        local = [rows_of.get(int(v), np.zeros(0, np.int64)) for v in V[:-1]]
        bptr = np.zeros(len(V), dtype=np.int64)
        bptr[1:] = np.cumsum([len(r) for r in local])
        bidx = pos[np.concatenate(local)] if local else np.zeros(0, np.int64)
        blocks[l] = dict(src_ids=V.astype(np.int32), indptr=bptr, indices=bidx.astype(np.int32),
                         rows=pos[nxt].astype(np.int32))
        nxt = V
    return blocks


def _layer0_input(features, blocks, indptr, indices, seeds, agg):
    """(table, indptr, indices, rows) of layer 0: the global table through the global CSR with rows = V_1, or, for the
    pools (their MLP runs on V_0's rows only), V_0's rows through block 0."""
    N = len(indptr) - 1
    if agg["type"] in ("maxpool", "meanpool"):
        b = blocks[0]
        return gather_clamped(features, b["src_ids"]), b["indptr"], b["indices"], b["rows"]
    v1 = blocks[1]["src_ids"] if len(blocks) > 1 else clamp_ids(seeds, N)
    return features, indptr, indices, v1


def block_embeddings(features, indptr, indices, aggregators, concat, seeds, normalize=True):
    """oracle.full_neighbor.full_neighbor_embeddings(node_ids=seeds) computed over csr_blocks: float32 [len(seeds), w]."""
    features = np.asarray(features, dtype=np.float32)
    L = len(aggregators)
    blocks = csr_blocks(indptr, indices, seeds, L)
    h = None
    for l, agg in enumerate(aggregators):
        act = (lambda x: x) if l == L - 1 else relu
        if l == 0:
            table, ptr, idx, rows = _layer0_input(features, blocks, indptr, indices, seeds, agg)
        else:
            table, ptr, idx, rows = h, blocks[l]["indptr"], blocks[l]["indices"], blocks[l]["rows"]
        h = layer(agg, table, ptr, idx, rows, concat, act)
    return l2_normalize(h) if normalize else h


def block_loss_grads(features, indptr, indices, aggregators, concat, node_ids, labels, pred_weights, pred_bias,
                     sigmoid_loss=False, weight_decay=0.0, identity_dim=0):
    """oracle.full_neighbor_grad.full_neighbor_loss_grads over csr_blocks: every layer runs in its block's local space
    (layer 0 on V_0's gathered rows through block 0), d(embeddings) is scattered from V_0 to [N+1, d].  Same returns."""
    features = np.asarray(features, dtype=np.float32)
    node_ids = np.asarray(node_ids, dtype=np.int64).reshape(-1)
    labels = np.asarray(labels, dtype=np.float64)
    L = len(aggregators)
    blocks = csr_blocks(indptr, indices, node_ids, L)
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
