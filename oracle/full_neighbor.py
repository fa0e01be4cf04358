"""Full-neighbourhood (layer-wise) inference: the contract of gs_csr_aggregate and of
SampleAndAggregate.full_neighbor_embeddings.  Plain numpy, fp32.

The sampled recursion of the reference (graphsage/models.py:300-330) computes, per layer, one aggregator call per hop
on sampled neighbour rows.  Layer-wise inference computes every node's layer-l row once over its WHOLE neighbourhood:

  h^0 = the model's source table [N+1, .] (row N the zero row; with identity_dim > 0 the embeddings come first);
  N(v) = v's CSR row; an empty row, and the dummy node N itself, use {N} (as the padded table does: isolated nodes and
         row N hold only the dummy id, graphsage/minibatch.py:227-245);
  layer l computes h^{l+1} for all N+1 rows, except the last, which computes only the requested node ids;
  mean     m = CSR_MEAN(h^l);                act(concat_or_add(h^l_v Ws, m_v Wn) + b)   aggregators.py:43-64
  gcn      m = CSR_MEAN_SELF(h^l);           act(m_v W + b)                               aggregators.py:101-116
  pools    z = relu(h^l Wm + bm) for all rows; p = CSR_MAX / CSR_MEAN(z);
                                             act(concat_or_add(h^l_v Ws, p_v Wn) + b)   aggregators.py:168-195, 246-273
  act = relu except on the last layer (identity, models.py:307-310); the result is l2-normalised (models.py:368).
With a d-regular graph and every num_samples = max_degree = d, the reference's sampler draws a permutation of each row,
so its sampled output equals this up to summation order (tests/golden/make_full_neighbor_golden.py).

gs_csr_aggregate, bit for bit: output row i is for node v = rows[i] (rows None: every node 0 .. n_nodes - 1, then the
dummy node n_nodes); its entries are indices[indptr[v] .. indptr[v+1]) in CSR order, an entry outside [0, R) reading
row R - 1 (R = table rows; gather.cu's clamp), and an empty row or a v outside [0, n_nodes) the row R - 1 alone.
  mean       acc = +0; acc = acc + x_j (fp32, in order); acc / fp32(count)        numerics.mean_f32 with k per row
  mean_self  the same, then acc = acc + x[clamp(v)]; acc / fp32(count + 1)
  max        m = x_0; m = fmax(m, x_j) in order                                  gs_segment_max

Test infrastructure - not imported by the product.
"""
import numpy as np

from .aggregate import l2_normalize, relu
from .numerics import gather_clamped

OPS = ("mean", "mean_self", "max")


def csr_rows(indptr, indices, n_src_rows, rows=None):
    """(nodes, entry lists): per output row, its node id and its source rows in CSR order (clamped; the dummy row for an
    empty row or a node outside [0, n_nodes))."""
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int64)
    n_nodes = len(indptr) - 1
    nodes = np.arange(n_nodes + 1) if rows is None else np.asarray(rows, dtype=np.int64).reshape(-1)
    inside = (nodes >= 0) & (nodes < n_nodes)
    safe = np.where(inside, nodes, 0)
    lo = np.where(inside, indptr[safe], 0)
    cnt = np.where(inside, np.maximum(indptr[np.minimum(safe + 1, n_nodes)] - lo, 0), 0)
    return nodes, lo, cnt


def csr_aggregate(table, indptr, indices, op, rows=None):
    """gs_csr_aggregate in the kernel's order, bit for bit.  table: float32 [R, F] or uint16 bf16 bits (widened exactly).
    Returns float32 [n, F]."""
    if op not in OPS:
        raise ValueError("op must be one of %s" % (OPS,))
    table = np.asarray(table)
    R = table.shape[0]
    indices = np.asarray(indices, dtype=np.int64)
    nodes, lo, cnt = csr_rows(indptr, indices, R, rows)
    n, F = len(nodes), table.shape[1]
    count = np.maximum(cnt, 1)

    def entry(sel, j):                             # source rows of entry j of the rows `sel`
        ids = np.full(len(sel), R - 1, dtype=np.int64)
        has = cnt[sel] > 0
        ids[has] = indices[lo[sel][has] + j]
        return gather_clamped(table, ids)

    acc = np.zeros((n, F), dtype=np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        if op == "max":
            acc = entry(np.arange(n), 0)
        start = 1 if op == "max" else 0
        for j in range(start, int(count.max()) if n else 0):
            sel = np.nonzero(count > j)[0]
            x = entry(sel, j)
            acc[sel] = np.fmax(acc[sel], x) if op == "max" else acc[sel] + x
        if op == "max":
            return acc
        if op == "mean_self":
            acc = acc + gather_clamped(table, nodes)
            return acc / (count + 1).astype(np.float32)[:, None]
        return acc / count.astype(np.float32)[:, None]


def dense_reference(table, indptr, indices, op, rows=None):
    """The same reduction in float64 from a dense adjacency-count matrix: the formula, not the order."""
    table = np.asarray(table, dtype=np.float64)
    R = table.shape[0]
    nodes, lo, cnt = csr_rows(indptr, indices, R, rows)
    indices = np.asarray(indices, dtype=np.int64)
    out = np.zeros((len(nodes), table.shape[1]))
    for i, (v, a, c) in enumerate(zip(nodes, lo, cnt)):
        ids = indices[a:a + c] if c else np.array([R - 1])
        ids = np.where((ids < 0) | (ids >= R), R - 1, ids)
        A = np.bincount(ids, minlength=R).astype(np.float64)           # one dense adjacency row (multiplicities)
        if op == "max":
            out[i] = table[ids].max(axis=0)
        elif op == "mean_self":
            A[v if 0 <= v < R else R - 1] += 1
            out[i] = A @ table / A.sum()
        else:
            out[i] = A @ table / A.sum()
    return out


def _combine(a, b, concat):
    return np.concatenate([a, b], axis=1) if concat else a + b


def layer(agg, h, indptr, indices, rows, concat, act):
    """One layer of the loop in the module docstring.  agg: {"type", weights...} as oracle.aggregate's dicts, plus
    "bias" when the aggregator has one."""
    kind = agg["type"]
    hs = h if rows is None else gather_clamped(h, rows)
    bias = agg.get("bias")
    if kind == "gcn":
        y = csr_aggregate(h, indptr, indices, "mean_self", rows) @ agg["weights"]
    else:
        if kind == "mean":
            p = csr_aggregate(h, indptr, indices, "mean", rows)
        elif kind in ("maxpool", "meanpool"):
            z = relu(h @ agg["mlp_weights"] + agg["mlp_bias"])
            p = csr_aggregate(z.astype(np.float32), indptr, indices, "max" if kind == "maxpool" else "mean", rows)
        else:
            raise ValueError(kind)
        y = _combine(hs @ agg["self_weights"], p @ agg["neigh_weights"], concat)
    if bias is not None:
        y = y + bias
    return act(y).astype(np.float32)


def full_neighbor_embeddings(features, indptr, indices, aggregators, concat, node_ids=None, normalize=True):
    """The layer loop: features [N+1, F] (row N zero), CSR over nodes 0..N-1, one aggregator dict per layer.  Returns
    float32 [len(node_ids) or N, out_w]."""
    h = np.asarray(features, dtype=np.float32)
    N = h.shape[0] - 1
    if len(indptr) != N + 1:
        raise ValueError("indptr must have N + 1 = %d entries" % (N + 1))
    node_ids = np.arange(N) if node_ids is None else np.asarray(node_ids, dtype=np.int64).reshape(-1)
    L = len(aggregators)
    for l, agg in enumerate(aggregators):
        last = l == L - 1
        h = layer(agg, h, indptr, indices, node_ids if last else None, concat, (lambda x: x) if last else relu)
    return l2_normalize(h) if normalize else h
